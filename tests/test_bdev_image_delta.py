"""Incremental volume images (oimgpu_bdev_image_track / _save_delta / _apply_delta, oim_b200/csrc/image_delta.cu; the
daemon's enable_bdev_image_tracking, save_bdev_image_delta and apply_bdev_image_delta; tools/oimcfg.py --track and
--deltas) compared with a numpy model of the delta format.

`model_delta` states the file a (parent, current) pair of stores must give: the 4096-byte header, the table of the
maximal runs of 4 KiB granules whose bytes differ from the parent's, split into zero runs and data runs, then the data
runs' bytes.  The format is canonical, so a save is compared with the model byte for byte.

CPU: the model on hand-built stores, the kernels' ptxas report, the struct layout, the C ABI's and the daemon's answers
without a GPU, oimcfg.py's command lines.  GPU (one H100): a base image and a chain of three deltas at block sizes 512,
520, 4096 and 4097, 2- and 4-way mirrors, every refusal, writes made by another process, a delta saved in the middle of
a VM's trace (launch per kick and resident poller), a daemon restart through oimcfg.py, and one 8 GiB volume."""
import base64
import errno
import glob
import json
import os
import re
import struct
import subprocess
import sys
import time

import numpy as np
import pytest

from oim_b200 import abi, build, lib, traces
from test_bdev_image import GRANULE, HEADER, UUID, _nbd_export, _read, _refused, content, model_digest, model_image
from test_daemon_mirror import IOSTAT, daemons, oracle_run, replica_digests, rpc, vm_trace  # noqa: F401
from test_mirror_replace import vm_run_split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAIL = struct.Struct("<IQQQ")       # reserved2, parent_digest[2], zero_bytes: bytes 100..127 of the header
ZERO_RUN = 1 << 63


# ---- the model ------------------------------------------------------------------------------------------------

def model_runs(parent, current):
    """the maximal runs of granules whose bytes differ from the parent's, split by kind -> [(offset, len, is_zero)]"""
    parent, current = np.asarray(parent, np.uint8), np.asarray(current, np.uint8)
    assert parent.size == current.size
    size = current.size
    ngran = (size + GRANULE - 1) // GRANULE
    p = np.zeros(ngran * GRANULE, np.uint8)
    c = np.zeros(ngran * GRANULE, np.uint8)
    p[:size], c[:size] = parent, current
    p, c = p.reshape(ngran, GRANULE), c.reshape(ngran, GRANULE)
    label = np.where((p != c).any(axis=1), np.where(c.any(axis=1), 2, 1), 0)      # 0 same, 1 now zero, 2 data
    edges = np.nonzero(np.diff(np.concatenate([[0], label, [0]])))[0]
    return [(int(s) * GRANULE, min(int(e) * GRANULE, size) - int(s) * GRANULE, bool(label[s] == 1))
            for s, e in zip(edges[:-1], edges[1:]) if label[s]]


def model_delta(parent, current, block_size, uuid=UUID) -> bytes:
    current = np.asarray(current, dtype=np.uint8)
    runs = model_runs(parent, current)
    data = b"".join(current[o:o + n].tobytes() for o, n, z in runs if not z)
    zero = sum(n for _, n, z in runs if z)
    d, pd = model_digest(current), model_digest(np.asarray(parent, np.uint8))
    head = HEADER.pack(b"OIMGPUDL", 1, block_size, current.size // block_size, GRANULE, 0, len(runs), len(data), d[0], d[1],
                       uuid.encode()) + TAIL.pack(0, pd[0], pd[1], zero)
    table = b"".join(struct.pack("<QQ", o, n | (ZERO_RUN if z else 0)) for o, n, z in runs)
    return head.ljust(4096, b"\0") + table.ljust((len(table) + 4095) // 4096 * 4096, b"\0") + data


def parse_delta(blob: bytes):
    """-> (header fields, runs [(offset, len, is_zero)]) of a delta"""
    magic, ver, bs, nb, gran, res, n, data_bytes, d0, d1, uuid = HEADER.unpack_from(blob)
    res2, p0, p1, zero = TAIL.unpack_from(blob, HEADER.size)
    runs = []
    for i in range(n):
        o, ln = struct.unpack_from("<QQ", blob, 4096 + 16 * i)
        runs.append((o, ln & ~ZERO_RUN, bool(ln & ZERO_RUN)))
    return {"magic": magic, "version": ver, "block_size": bs, "num_blocks": nb, "granule_bytes": gran, "reserved": res,
            "nextents": n, "data_bytes": data_bytes, "digest": (d0, d1), "uuid": uuid.decode().rstrip("\0"),
            "reserved2": res2, "parent_digest": (p0, p1), "zero_bytes": zero}, runs


def apply_model(parent, blob):
    """the store a delta makes of `parent`"""
    h, runs = parse_delta(blob)
    s = np.array(parent, dtype=np.uint8)
    pos = 4096 + (16 * h["nextents"] + 4095) // 4096 * 4096
    for o, n, z in runs:
        if z:
            s[o:o + n] = 0
        else:
            s[o:o + n] = np.frombuffer(blob, np.uint8, n, pos)
            pos += n
    assert pos == len(blob)
    return s


def mutate(s, seed):
    """the next state of a store: granules turned to zero, turned non-zero, changed in a few bytes, a zero granule next to
    a new data granule, and the last byte of the store flipped; everything else keeps its bytes"""
    rng = np.random.default_rng(seed)
    s = s.copy()
    ngran = (s.size + GRANULE - 1) // GRANULE
    nz = [g for g in range(ngran) if s[g * GRANULE:(g + 1) * GRANULE].any()]
    zs = [g for g in range(ngran) if not s[g * GRANULE:(g + 1) * GRANULE].any()]
    for g in rng.choice(nz, size=min(len(nz), 3), replace=False) if nz else []:
        s[g * GRANULE:(g + 1) * GRANULE] = 0
    for g in rng.choice(zs, size=min(len(zs), 3), replace=False) if zs else []:
        s[g * GRANULE + int(rng.integers(0, GRANULE - 8)):][:8] = rng.integers(1, 256, size=8, dtype=np.uint8)
    for _ in range(4):
        pos = int(rng.integers(0, s.size))
        s[pos] = (int(s[pos]) + 1 + int(rng.integers(0, 254))) % 256
    g = int(rng.integers(0, max(1, ngran - 1)))
    s[g * GRANULE:(g + 1) * GRANULE] = 0
    s[(g + 1) * GRANULE:(g + 1) * GRANULE + 1] = 0x33
    s[-1] ^= 0x81
    return s


def test_model_runs_are_maximal_and_split_by_kind():
    p = np.zeros(12 * GRANULE, dtype=np.uint8)
    p[1 * GRANULE] = p[2 * GRANULE] = p[6 * GRANULE] = p[9 * GRANULE] = 1
    c = p.copy()
    c[1 * GRANULE] = 0                      # granule 1 now zero
    c[2 * GRANULE] = 0                      # granule 2 too: one zero run of two
    c[3 * GRANULE + 7] = 5                  # granule 3 now data: touches the zero run
    c[4 * GRANULE] = 9                      # granule 4 too: one data run of two
    c[6 * GRANULE] = 1                      # granule 6 rewritten with the same bytes: not in the delta
    c[9 * GRANULE + 1] = 2                  # granule 9 changed, still data
    c[11 * GRANULE] = 4                     # the last granule
    assert model_runs(p, c) == [(GRANULE, 2 * GRANULE, True), (3 * GRANULE, 2 * GRANULE, False),
                                (9 * GRANULE, GRANULE, False), (11 * GRANULE, GRANULE, False)]
    blob = model_delta(p, c, 512)
    assert len(blob) == 4096 + 4096 + 4 * GRANULE
    h, runs = parse_delta(blob)
    assert (h["nextents"], h["data_bytes"], h["zero_bytes"]) == (4, 4 * GRANULE, 2 * GRANULE)
    assert h["digest"] == model_digest(c) and h["parent_digest"] == model_digest(p)
    assert (apply_model(p, blob) == c).all()


@pytest.mark.parametrize("bs,nb", [(520, 17), (4097, 3)])
def test_model_partial_last_granule(bs, nb):
    """a store whose size is not a multiple of 4096: the last run, of either kind, ends at the end of the store"""
    size = bs * nb
    assert size % GRANULE
    last = (size - 1) // GRANULE * GRANULE
    p = np.zeros(size, dtype=np.uint8)
    c = p.copy()
    c[-1] = 7
    assert model_runs(p, c) == [(last, size - last, False)]
    assert model_runs(c, p) == [(last, size - last, True)]
    blob = model_delta(c, p, bs)
    assert len(blob) == 8192 and (apply_model(c, blob) == p).all()
    c2 = content("dense", nb, bs, 1)
    assert (apply_model(p, model_delta(p, c2, bs)) == c2).all()


def test_model_unchanged_store_gives_an_empty_delta():
    s = content("sparse", 100, 512, 3)
    blob = model_delta(s, s, 512)
    h, runs = parse_delta(blob)
    assert len(blob) == 4096 and runs == [] and h["data_bytes"] == h["zero_bytes"] == 0
    assert h["digest"] == h["parent_digest"] == model_digest(s)


def test_model_chain_reaches_the_last_state():
    s = [content("sparse", 300, 520, 4)]
    for k in range(3):
        s.append(mutate(s[-1], k))
    cur = s[0]
    for a, b in zip(s, s[1:]):
        cur = apply_model(cur, model_delta(a, b, 520))
    assert (cur == s[-1]).all()


# ---- CPU: the kernels, the C ABI, the daemon and oimcfg.py without a GPU ------------------------------------------

KERNELS = ("oim_image_delta_scan_kernel", "oim_image_delta_zero_kernel")


def test_delta_kernels_compile_for_sm90a_without_spills(tmp_path):
    src = os.path.join(ROOT, "oim_b200", "csrc", "image_delta.cu")
    r = subprocess.run([build.NVCC, *[f for f in build.FLAGS if f != "-shared"], "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "image_delta.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for k in KERNELS:
        m = re.search(rf"Compiling entry function '(\S*{k}\S*)' for 'sm_90a'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads", r.stderr, re.S)
        assert m and m.group(2) == "0" and m.group(3) == "0" and m.group(4) == "0", (k, r.stderr[-3000:])
    sass = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", build.build()], capture_output=True, text=True).stdout
    for k in KERNELS:
        assert re.search(rf"Function : \S*{k}", sass), k


def test_delta_info_struct_matches_c(tmp_path):
    probe = tmp_path / "probe.c"
    fields = ("nextents", "data_bytes", "zero_bytes", "file_bytes", "parent_digest", "digest", "block_size",
              "granule_bytes", "uuid")
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "oimgpu.h"\n'
                     "#define O(f) offsetof(struct oimgpu_image_delta_info, f)\n"
                     'int main(void){printf("%zu' + " %zu" * len(fields) + '\\n",sizeof(struct oimgpu_image_delta_info),'
                     + ",".join(f"O({f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(probe), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    d = abi.image_delta_info_dtype
    assert got == [d.itemsize] + [d.fields[f][1] for f in fields]


def test_delta_abi_without_gpu(tmp_path):
    L = lib.load()
    out = np.zeros(1, dtype=abi.image_delta_info_dtype)
    p = str(tmp_path / "x.delta").encode()
    for fn in (L.oimgpu_bdev_image_save_delta, L.oimgpu_bdev_image_apply_delta):
        assert fn(None, p, out.ctypes.data) == -errno.EINVAL
        assert fn(b"x", None, out.ctypes.data) == -errno.EINVAL
        assert fn(b"x", p, None) == -errno.EINVAL
    assert L.oimgpu_bdev_image_track(None, 1) == -errno.EINVAL
    if glob.glob("/dev/nvidia[0-9]*"):
        return      # below: a library that never found a GPU
    assert L.oimgpu_bdev_image_track(b"x", 1) == -errno.ENODEV
    assert L.oimgpu_init_control_only() == 0
    try:
        name = lib.construct_malloc_bdev(64, 512, name="CtlDelta")
        for nm in (name, "nope"):
            assert L.oimgpu_bdev_image_track(nm.encode(), 1) == -errno.ENODEV
            for fn in (L.oimgpu_bdev_image_save_delta, L.oimgpu_bdev_image_apply_delta):
                assert fn(nm.encode(), p, out.ctypes.data) == -errno.ENODEV
    finally:
        lib.fini()
    assert not os.path.exists(p)


def test_delta_methods_without_a_gpu(daemons, tmp_path):
    s = daemons("ours", ["--control-only"])
    rpc(s, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512, "name": "V"})
    nodev = {"code": -32602, "message": "No such device"}
    bad = {"code": -32602, "message": "Invalid parameters"}
    for p in ({"name": "V"}, {"name": "V", "enable": False}, {"name": "nope"}):
        assert rpc(s, "enable_bdev_image_tracking", p) == {"error": nodev}, p
    for p in ({}, {"enable": True}, {"name": 1}, {"name": "V", "enable": 1}, {"name": "V", "x": 1}, None):
        assert rpc(s, "enable_bdev_image_tracking", p) == {"error": bad}, p
    for m in ("save_bdev_image_delta", "apply_bdev_image_delta"):
        for p in ({"name": "V", "path": str(tmp_path / "v.delta")}, {"name": "nope", "path": str(tmp_path / "n.delta")}):
            assert rpc(s, m, p) == {"error": nodev}, (m, p)
        for p in ({}, {"name": "V"}, {"path": "/x"}, {"name": 1, "path": "/x"}, {"name": "V", "path": 2},
                  {"name": "V", "path": "/x", "x": 1}, None):
            assert rpc(s, m, p) == {"error": bad}, (m, p)
    # the image methods still take exactly their two keys
    assert rpc(s, "save_bdev_image", {"name": "V", "path": "/x", "track": True}) == {"error": bad}
    assert not os.listdir(tmp_path)
    cfg = rpc(s, "get_subsystem_config", {"name": "bdev"})
    assert [x["method"] for x in cfg] == ["set_bdev_options", "construct_malloc_bdev"]


def test_oimcfg_command_lines():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import oimcfg
    ok = {("save", "s"): ("save", "s", None, False, []), ("load", "s"): ("load", "s", None, False, []),
          ("save", "s", "--images", "d"): ("save", "s", "d", False, []),
          ("load", "s", "--images", "d"): ("load", "s", "d", False, []),
          ("save", "s", "--images", "d", "--track"): ("save", "s", "d", True, []),
          ("save", "s", "--deltas", "x"): ("save", "s", None, False, ["x"]),
          ("load", "s", "--images", "d", "--deltas", "a", "b"): ("load", "s", "d", False, ["a", "b"])}
    for args, want in ok.items():
        assert oimcfg.parse(list(args)) == want, args
    for args in (["save"], ["x", "s"], ["save", "s", "--images"], ["save", "s", "--track"], ["load", "s", "--deltas", "a"],
                 ["save", "s", "--deltas", "a", "b"], ["load", "s", "--images", "d", "--track"], ["save", "s", "extra"]):
        assert oimcfg.parse(args) is None, args


# ---- GPU ----------------------------------------------------------------------------------------------------

def _info_of(blob):
    h, _ = parse_delta(blob)
    return {"num_blocks": h["num_blocks"], "block_size": h["block_size"], "granule_bytes": GRANULE, "nextents": h["nextents"],
            "data_bytes": h["data_bytes"], "zero_bytes": h["zero_bytes"], "file_bytes": len(blob),
            "parent_digest": h["parent_digest"], "digest": h["digest"], "uuid": h["uuid"]}


CHAIN = [512, 4096, 520, 4097]


@pytest.mark.gpu
@pytest.mark.parametrize("bs", CHAIN, ids=[f"bs{b}" for b in CHAIN])
def test_chain_of_deltas_matches_the_model(gpu, tmp_path, bs):
    """a base image, then three deltas, each written over the whole store (unchanged granules rewritten with their own
    bytes); a fresh bdev loaded from the image and given the deltas in order ends equal to the source"""
    nb = 2000 if bs < 4096 else 700
    states = [content("sparse", nb, bs, seed=bs)]
    for k in range(3):
        states.append(mutate(states[-1], bs + k))
    src = gpu.construct_malloc_bdev(nb, bs, name=f"csrc{bs}", uuid=UUID, device=0)
    dst = gpu.construct_malloc_bdev(nb, bs, name=f"cdst{bs}", device=0)
    try:
        gpu.bdev_write_raw(src, 0, states[0])
        gpu.bdev_image_track(src)
        gpu.bdev_image_track(src)               # enabling twice is harmless
        gpu.bdev_image_save(src, tmp_path / "base.img")
        assert _read(tmp_path / "base.img") == model_image(states[0], bs), "a tracked save wrote another image"
        for k in (1, 2, 3):
            gpu.bdev_write_raw(src, 0, states[k])
            info = gpu.bdev_image_save_delta(src, tmp_path / f"d{k}.delta")
            got, want = _read(tmp_path / f"d{k}.delta"), model_delta(states[k - 1], states[k], bs)
            assert len(got) == len(want) and got[:4096] == want[:4096], f"delta {k}: header differs from the model's"
            assert got == want, f"delta {k}: table or data differs from the model's"
            assert info == _info_of(want)
            assert info["zero_bytes"] > 0 and info["data_bytes"] > 0
        info = gpu.bdev_image_save_delta(src, tmp_path / "d4.delta")
        assert _read(tmp_path / "d4.delta") == model_delta(states[3], states[3], bs) and info["file_bytes"] == 4096
        gpu.bdev_image_load(dst, tmp_path / "base.img")
        for k in (1, 2, 3, 4):
            info = gpu.bdev_image_apply_delta(dst, tmp_path / f"d{k}.delta")
            assert info["digest"] == model_digest(states[min(k, 3)])
            if (nb * bs) % 8 == 0:
                assert gpu.bdev_digest(dst) == model_digest(states[min(k, 3)])
        assert (gpu.bdev_read_raw(dst, 0, nb * bs) == states[3]).all()
    finally:
        gpu.delete_bdev(src)
        gpu.delete_bdev(dst)


@pytest.mark.gpu
@pytest.mark.parametrize("nrep", [2, 4])
def test_mirrors_take_a_delta_in_every_replica(gpu, tmp_path, nrep):
    nb, bs = 1500, 4096
    s0 = content("sparse", nb, bs, seed=nrep)
    s1 = mutate(s0, nrep)
    s2 = mutate(s1, nrep + 1)
    src = gpu.construct_malloc_bdev(nb, bs, name=f"mdsrc{nrep}", uuid=UUID, device=0)
    dst = gpu.construct_mirror_bdev(nb, bs, [0] * nrep, name=f"mddst{nrep}")
    try:
        gpu.bdev_write_raw(src, 0, s0)
        gpu.bdev_image_track(src)
        gpu.bdev_image_save(src, tmp_path / "base.img")
        for k, s in ((1, s1), (2, s2)):
            gpu.bdev_write_raw(src, 0, s)
            gpu.bdev_image_save_delta(src, tmp_path / f"d{k}.delta")
        for r in range(nrep):
            gpu.bdev_write_raw(dst, 0, np.full(nb * bs, 0x77, dtype=np.uint8), replica=r)
        gpu.bdev_image_load(dst, tmp_path / "base.img")
        gpu.bdev_image_apply_delta(dst, tmp_path / "d1.delta")
        for r in range(nrep):
            assert gpu.bdev_digest(dst, r) == model_digest(s1), f"replica {r}"
        # replica 1 drifts: the mirror must not take the next delta, and nothing changes
        gpu.bdev_write_raw(dst, 5 * bs, np.full(bs, 0xEE, dtype=np.uint8), replica=1)
        before = [gpu.bdev_digest(dst, r) for r in range(nrep)]
        _refused(lambda: gpu.bdev_image_apply_delta(dst, tmp_path / "d2.delta"), -errno.ESTALE)
        assert [gpu.bdev_digest(dst, r) for r in range(nrep)] == before
        gpu.mirror_check(dst, repair=True)
        gpu.bdev_image_apply_delta(dst, tmp_path / "d2.delta")
        for r in range(nrep):
            assert gpu.bdev_digest(dst, r) == model_digest(s2), f"replica {r}"
    finally:
        gpu.delete_bdev(src)
        gpu.delete_bdev(dst)


@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_delta_refusals(gpu, tmp_path):
    nb, bs = 1000, 512
    s0 = content("sparse", nb, bs, seed=9)
    s1 = mutate(s0, 1)
    s2 = mutate(s1, 2)
    name = gpu.construct_malloc_bdev(nb, bs, name="drefuse", uuid=UUID, device=0)
    dst = gpu.construct_malloc_bdev(nb, bs, name="drefuse-dst", device=0)
    other = gpu.construct_malloc_bdev(nb + 1, bs, name="drefuse-geo", device=0)
    try:
        gpu.bdev_write_raw(name, 0, s0)
        # no tracking, then no baseline yet
        _refused(lambda: gpu.bdev_image_save_delta(name, tmp_path / "u.delta"), -errno.ENODATA)
        gpu.bdev_image_track(name)
        _refused(lambda: gpu.bdev_image_save_delta(name, tmp_path / "u.delta"), -errno.ENODATA)
        _refused(lambda: gpu.bdev_image_track("nope"), -errno.ENODEV)
        gpu.bdev_image_save(name, tmp_path / "base.img")
        gpu.bdev_write_raw(name, 0, s1)
        gpu.bdev_image_save_delta(name, tmp_path / "d1.delta")
        gpu.bdev_write_raw(name, 0, s2)
        # a failed save (EEXIST) keeps the baseline: the next delta is still taken against s1
        _refused(lambda: gpu.bdev_image_save_delta(name, tmp_path / "d1.delta"), -errno.EEXIST)
        assert _read(tmp_path / "d1.delta") == model_delta(s0, s1, bs)
        _refused(lambda: gpu.bdev_image_save_delta(name, tmp_path / "no-dir" / "x.delta"), -errno.ENOENT)
        # save: not while an NBD export or a bio channel serves the bdev
        sock, th, rc = _nbd_export(gpu, name)
        try:
            _refused(lambda: gpu.bdev_image_save_delta(name, tmp_path / "nbd.delta"), -errno.EBUSY)
        finally:
            sock.close()
            th.join(20)
        assert rc == [0]
        with gpu.BioChan(name):
            _refused(lambda: gpu.bdev_image_save_delta(name, tmp_path / "bio.delta"), -errno.EBUSY)
        assert not os.path.exists(tmp_path / "nbd.delta") and not os.path.exists(tmp_path / "bio.delta")
        gpu.bdev_image_save_delta(name, tmp_path / "d2.delta")
        assert _read(tmp_path / "d2.delta") == model_delta(s1, s2, bs)
        # apply: out of order, or onto the wrong base, leaves the bdev as it was
        gpu.bdev_image_load(dst, tmp_path / "base.img")
        d0 = gpu.bdev_digest(dst)
        _refused(lambda: gpu.bdev_image_apply_delta(dst, tmp_path / "d2.delta"), -errno.ESTALE)
        assert gpu.bdev_digest(dst) == d0
        _refused(lambda: gpu.bdev_image_apply_delta(other, tmp_path / "d1.delta"), -errno.EINVAL)     # geometry
        with gpu.BioChan(dst):
            _refused(lambda: gpu.bdev_image_apply_delta(dst, tmp_path / "d1.delta"), -errno.EBUSY)
        # malformed deltas are refused before a store is touched
        blob = _read(tmp_path / "d1.delta")
        h, runs = parse_delta(blob)
        assert len(runs) >= 4 and any(z for _, _, z in runs) and any(not z for _, _, z in runs)

        def variant(tag, b):
            p = tmp_path / f"{tag}.delta"
            p.write_bytes(bytes(b))
            return p

        def entry(b, i, o, ln):
            b[4096 + 16 * i:4096 + 16 * i + 16] = struct.pack("<QQ", o, ln)
            return b
        o0, n0, z0 = runs[0]
        o1, n1, z1 = runs[1]
        raw1 = n1 | (ZERO_RUN if z1 else 0)
        bad = [variant("magic", b"OIMGPUIM" + blob[8:]), variant("version", blob[:8] + struct.pack("<I", 2) + blob[12:]),
               variant("reserved2", blob[:100] + struct.pack("<I", 1) + blob[104:]),
               variant("short", blob[:-1]), variant("long", blob + b"\0"), variant("header-only", blob[:100]),
               variant("overlap", entry(bytearray(blob), 1, o0, raw1)),
               variant("unaligned", entry(bytearray(blob), 1, o1 + 8, raw1)),
               variant("range", entry(bytearray(blob), 1, nb * bs // GRANULE * GRANULE + GRANULE, raw1)),
               variant("kind", entry(bytearray(blob), 1, o1, n1 | (0 if z1 else ZERO_RUN))),
               variant("high-bits", entry(bytearray(blob), 1, o1, raw1 | 1 << 62)),
               variant("header-padding", blob[:200] + b"\1" + blob[201:]),
               variant("table-padding", blob[:8191] + b"\1" + blob[8192:])]
        assert 16 * len(runs) < 4096, "the table has no padding to tamper with"
        # a run moved down to touch the run before it, of its own kind
        same = [i for i in range(1, len(runs)) if runs[i][2] == runs[i - 1][2]]
        assert same, runs
        i = same[0]
        bad.append(variant("same-kind-touching", entry(bytearray(blob), i, runs[i - 1][0] + runs[i - 1][1],
                                                       runs[i][1] | (ZERO_RUN if runs[i][2] else 0))))
        for p in bad:
            _refused(lambda: gpu.bdev_image_apply_delta(dst, p), -errno.EINVAL)
            assert gpu.bdev_digest(dst) == d0, f"{p.name}: the bdev changed"
        # a delta is not an image
        _refused(lambda: gpu.bdev_image_load(dst, tmp_path / "d1.delta"), -errno.EINVAL)
        assert gpu.bdev_digest(dst) == d0
        gpu.bdev_image_apply_delta(dst, tmp_path / "d1.delta")
        gpu.bdev_image_apply_delta(dst, tmp_path / "d2.delta")
        assert (gpu.bdev_read_raw(dst, 0, nb * bs) == s2).all()
        # a flipped data byte is applied and caught by the digest; the tracked bdev's baseline is then gone
        gpu.bdev_image_track(dst)
        gpu.bdev_image_load(dst, tmp_path / "base.img")
        b = bytearray(blob)
        b[-1] ^= 0x10
        _refused(lambda: gpu.bdev_image_apply_delta(dst, variant("flipped", b)), -errno.EIO)
        _refused(lambda: gpu.bdev_image_save_delta(dst, tmp_path / "after-eio.delta"), -errno.ENODATA)
        # disabling drops the tables and the baseline; enabling again starts without one
        gpu.bdev_image_track(name, False)
        _refused(lambda: gpu.bdev_image_save_delta(name, tmp_path / "off.delta"), -errno.ENODATA)
        gpu.bdev_image_track(name)
        _refused(lambda: gpu.bdev_image_save_delta(name, tmp_path / "off.delta"), -errno.ENODATA)
        assert not os.path.exists(tmp_path / "off.delta") and not os.path.exists(tmp_path / "after-eio.delta")
    finally:
        for nm in (name, dst, other):
            gpu.delete_bdev(nm)


EFBIG_SCRIPT = r"""
import json, os, resource, signal, sys
import numpy as np
sys.path.insert(0, os.getcwd())
from oim_b200 import lib
d, bs = sys.argv[1], int(sys.argv[2])
s = [np.load(os.path.join(d, f"s{k}.npy")) for k in range(3)]
lib.init([0])
out = {}
try:
    name = lib.construct_malloc_bdev(s[0].size // bs, bs, name="efbig", uuid=sys.argv[3], device=0)
    lib.bdev_write_raw(name, 0, s[0])
    lib.bdev_image_track(name)
    lib.bdev_image_save(name, os.path.join(d, "base.img"))
    signal.signal(signal.SIGXFSZ, signal.SIG_IGN)
    soft, hard = resource.getrlimit(resource.RLIMIT_FSIZE)

    def limited(fn, path):
        # files of this process may not grow past their header and table: the data write fails, after the scan
        resource.setrlimit(resource.RLIMIT_FSIZE, (8192, hard))
        try:
            fn(name, path)
            return 0
        except lib.OimGpuError as e:
            return e.rc
        finally:
            resource.setrlimit(resource.RLIMIT_FSIZE, (soft, hard))
    lib.bdev_write_raw(name, 0, s[1])
    out["delta"] = limited(lib.bdev_image_save_delta, os.path.join(d, "fail.delta"))
    lib.bdev_image_save_delta(name, os.path.join(d, "d1.delta"))
    lib.bdev_write_raw(name, 0, s[2])
    out["image"] = limited(lib.bdev_image_save, os.path.join(d, "fail.img"))
    lib.bdev_image_save_delta(name, os.path.join(d, "d2.delta"))
finally:
    lib.fini()
print(json.dumps(out))
"""


@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_save_failing_after_the_scan_keeps_the_baseline(gpu, tmp_path):
    """A delta save and a tracked image save whose data write fails (EFBIG under a file size limit) after the scan has
    rewritten the spare fingerprint table: the file is removed and the next delta is still taken against the old
    baseline.  Run in a process of its own, the only one the size limit applies to."""
    nb, bs = 1000, 4096
    s = [content("sparse", nb, bs, seed=31)]
    s += [mutate(s[0], 32)]
    s += [mutate(s[1], 33)]
    for k, x in enumerate(s):
        np.save(tmp_path / f"s{k}.npy", x)
    r = subprocess.run([sys.executable, "-c", EFBIG_SCRIPT, str(tmp_path), str(bs), UUID], cwd=ROOT, capture_output=True,
                       text=True, timeout=150)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out == {"delta": -errno.EFBIG, "image": -errno.EFBIG}, out
    assert not os.path.exists(tmp_path / "fail.delta") and not os.path.exists(tmp_path / "fail.img")
    assert _read(tmp_path / "d1.delta") == model_delta(s[0], s[1], bs), "a failed delta save moved the baseline"
    assert _read(tmp_path / "d2.delta") == model_delta(s[1], s[2], bs), "a failed image save moved the baseline"


def _hex(d):
    return f"{d[0]:016x}{d[1]:016x}"


@pytest.mark.gpu
@pytest.mark.timeout(180)
def test_delta_methods_and_writes_of_another_process(gpu, daemons, tmp_path):
    """the daemon tracks A and saves its base image; this process then writes A's store through an imported replica,
    which no session of the daemon sees, and the daemon's next delta holds exactly those writes"""
    nb, bs = 4096, 4096
    s0 = content("sparse", nb, bs, seed=21)
    s1 = mutate(s0, 22)
    d = daemons("ours", ["--gpus", "0"])
    assert rpc(d, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "A", "uuid": UUID}) == "A"
    assert rpc(d, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "B"}) == "B"

    def write(s):
        local = gpu.construct_mirror_bdev_remote(nb, bs, 0, [base64.b64decode(rpc(d, "export_bdev_store", {"name": "A"}))],
                                                 name="A-writer")
        try:
            gpu.bdev_write_raw(local, 0, s, replica=1)
        finally:
            gpu.delete_bdev(local)
    write(s0)
    assert rpc(d, "enable_bdev_image_tracking", {"name": "A"}) is True
    assert rpc(d, "enable_bdev_image_tracking", {"name": "A", "enable": True}) is True
    base, path = str(tmp_path / "a.img"), str(tmp_path / "a1.delta")
    assert rpc(d, "save_bdev_image", {"name": "A", "path": base})["file_bytes"] == len(model_image(s0, bs))
    write(s1)
    want = model_delta(s0, s1, bs)
    h, runs = parse_delta(want)
    shape = {"name": "A", "path": path, "block_size": bs, "num_blocks": nb, "uuid": UUID, "extents": len(runs),
             "data_bytes": h["data_bytes"], "zero_bytes": h["zero_bytes"], "file_bytes": len(want),
             "parent_digest": _hex(model_digest(s0)), "digest": _hex(model_digest(s1))}
    assert rpc(d, "save_bdev_image_delta", {"name": "A", "path": path}) == shape
    assert _read(path) == want
    assert rpc(d, "save_bdev_image_delta", {"name": "A", "path": path}) == {"error": {"code": -32602, "message": "File exists"}}
    assert rpc(d, "save_bdev_image_delta", {"name": "B", "path": path + ".b"}) == \
        {"error": {"code": -32602, "message": "No data available"}}
    assert rpc(d, "load_bdev_image", {"name": "B", "path": base})["name"] == "B"
    assert rpc(d, "apply_bdev_image_delta", {"name": "B", "path": path}) == {**shape, "name": "B"}
    assert replica_digests(gpu, d, "B", 1, nb, bs) == [model_digest(s1)]
    assert rpc(d, "apply_bdev_image_delta", {"name": "B", "path": path}) == \
        {"error": {"code": -32602, "message": "Stale file handle"}}
    assert rpc(d, "enable_bdev_image_tracking", {"name": "A", "enable": False}) is True
    assert rpc(d, "save_bdev_image_delta", {"name": "A", "path": path + ".off"}) == \
        {"error": {"code": -32602, "message": "No data available"}}
    assert rpc(d, "construct_vhost_scsi_controller", {"ctrlr": "scsi0"}) is True
    assert rpc(d, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 0, "bdev_name": "B"}) == 0
    cfg = rpc(d, "get_subsystem_config", {"name": "bdev"}) + rpc(d, "get_subsystem_config", {"name": "vhost"})
    assert not [x for x in cfg if "image" in x["method"]]


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("mode,bs", [("kick", 512), ("poller", 4096)])
def test_delta_in_the_middle_of_a_vm(gpu, oracles, daemons, tmp_path, mode, bs):
    """the volume is tracked and imaged empty; a delta saved between the two halves of a VM's trace is the model's
    delta from empty to the volume at that point (its digest is the store's, read right after), and the second half
    then completes as the C restatement computes for the whole trace"""
    seed = 900 + bs
    rq_by_q, nb = vm_trace(bs, 1, seed)
    rq = rq_by_q[0]
    a = daemons("a", ["--gpus", "0"] + (["--poller"] if mode == "poller" else []))
    assert rpc(a, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "Vol", "uuid": UUID}) == "Vol"
    assert rpc(a, "enable_bdev_image_tracking", {"name": "Vol"}) is True
    assert rpc(a, "save_bdev_image", {"name": "Vol", "path": str(tmp_path / "base.img")})["extents"] == 0
    assert rpc(a, "construct_vhost_scsi_controller", {"ctrlr": "scsi0"}) is True
    assert rpc(a, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 0, "bdev_name": "Vol"}) == 0
    done = []

    def between():
        rep = rpc(a, "save_bdev_image_delta", {"name": "Vol", "path": str(tmp_path / "mid.delta")})
        assert rep["name"] == "Vol" and rep["uuid"] == UUID, rep
        done.append((rep, rpc(a, "get_bdevs_iostat", {"name": "Vol"})[1], replica_digests(gpu, a, "Vol", 1, nb, bs)[0]))
    img, mem, used = vm_run_split(a, rq, seed, between)
    assert done, "the delta was not saved"
    rep, stat, digest = done[0]
    blob = _read(tmp_path / "mid.delta")
    empty = np.zeros(nb * bs, np.uint8)
    store = apply_model(empty, blob)
    assert blob == model_delta(empty, store, bs), "the delta is not the model's"
    h, _ = parse_delta(blob)
    assert h["digest"] == digest == model_digest(store), "the delta is not the volume between the two halves"
    assert rep["file_bytes"] == len(blob) and rep["extents"] == h["nextents"] and rep["digest"] == _hex(digest)
    assert 0 < stat["num_write_ops"] + stat["num_read_ops"], "the delta came before any request"
    wimg, wused, wstore, wstat = oracle_run(oracles, [rq], nb, bs, seed)
    assert used == wused, "used elements differ from the checker's"
    deadline = time.time() + 10
    while True:
        st = rpc(a, "get_bdevs_iostat", {"name": "Vol"})[1]
        got = {k: st[k] for k in IOSTAT}
        if got == {k: wstat[k] for k in IOSTAT} or time.time() > deadline:
            break
        time.sleep(0.05)
    assert got == {k: wstat[k] for k in IOSTAT}, "the delta was counted, or the second half was not served"
    assert replica_digests(gpu, a, "Vol", 1, nb, bs) == [gpu.digest_host(wstore)]
    local = gpu.construct_malloc_bdev(nb, bs, name="mid-copy", device=0)
    try:
        gpu.bdev_image_load(local, tmp_path / "base.img")
        gpu.bdev_image_apply_delta(local, tmp_path / "mid.delta")
        assert gpu.bdev_digest(local) == digest
    finally:
        gpu.delete_bdev(local)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_restart_through_oimcfg_deltas(gpu, daemons, tmp_path):
    """oimcfg.py save --images --track, writes, save --deltas twice, the daemon stops, a fresh one starts, oimcfg.py load
    --images --deltas: every bdev - a plain volume, a 2-way mirror and an empty volume - has its old digests and listing"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import oimcfg
    nb, bs = 4096, 4096
    old = daemons("old", ["--gpus", "0"])
    assert rpc(old, "construct_malloc_bdev", {"num_blocks": nb, "block_size": bs, "name": "plain", "uuid": UUID}) == "plain"
    assert rpc(old, "construct_mirror_bdev", {"num_blocks": nb, "block_size": 520 * 8, "name": "mir", "replicas": 2}) == "mir"
    assert rpc(old, "construct_malloc_bdev", {"num_blocks": 64, "block_size": 512, "name": "empty"}) == "empty"
    assert rpc(old, "construct_vhost_scsi_controller", {"ctrlr": "scsi0"}) is True
    assert rpc(old, "add_vhost_scsi_lun", {"ctrlr": "scsi0", "scsi_target_num": 0, "bdev_name": "plain"}) == 0
    state = {"plain": np.zeros(nb * bs, np.uint8), "mir": np.zeros(nb * bs, np.uint8)}

    def write(step):
        for nm, seed in (("plain", 1), ("mir", 2)):
            state[nm] = content("sparse", nb, 4096, seed) if step == 0 else mutate(state[nm], 10 * step + seed)
            local = gpu.construct_mirror_bdev_remote(nb, 4096, 0, [base64.b64decode(rpc(old, "export_bdev_store", {"name": nm}))],
                                                     name="writer")
            try:
                gpu.bdev_write_raw(local, 0, state[nm], replica=1)
            finally:
                gpu.delete_bdev(local)
        rpc(old, "check_mirror_bdev", {"name": "mir", "repair": True})
    write(0)
    images = tmp_path / "images"
    images.mkdir()
    saved = oimcfg.save(oimcfg.Rpc(old.rpc), str(images), track=True)
    dirs = []
    for step in (1, 2):
        write(step)
        dirs.append(tmp_path / f"d{step}")
        dirs[-1].mkdir()
        oimcfg.save(oimcfg.Rpc(old.rpc), deltas=str(dirs[-1]))
        assert sorted(os.listdir(dirs[-1])) == ["empty.delta", "mir.delta", "plain.delta"]
    assert os.path.getsize(dirs[-1] / "empty.delta") == 4096
    listing = rpc(old, "get_bdevs")
    digests = {b["name"]: replica_digests(gpu, old, b["name"], len(b.get("driver_specific", {}).get("mirror", {}).get("replicas", [0])),
                                          b["num_blocks"], b["block_size"]) for b in listing}
    assert digests["plain"] == [model_digest(state["plain"])]
    old.close()
    fresh = daemons("fresh", ["--gpus", "0"])
    oimcfg.load(oimcfg.Rpc(fresh.rpc), saved, str(images), [str(p) for p in dirs])
    assert rpc(fresh, "get_bdevs") == listing
    for b in listing:
        n = len(b.get("driver_specific", {}).get("mirror", {}).get("replicas", [0]))
        assert replica_digests(gpu, fresh, b["name"], n, b["num_blocks"], b["block_size"]) == digests[b["name"]], b["name"]
    assert [c["backend_specific"]["scsi"][0]["luns"][0]["bdev_name"] for c in rpc(fresh, "get_vhost_controllers")] == ["plain"]


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_eight_gib_volume_delta(gpu, tmp_path):
    """500 scattered granules and a 48 MiB region rewritten after the base image: data_bytes is exactly their
    granules, and the delta applied to the base image gives the source's digest"""
    nb, bs = 2 << 20, 4096
    size = nb * bs
    rng = np.random.default_rng(8)
    src = gpu.construct_malloc_bdev(nb, bs, name="dbig", uuid=UUID, device=0)
    dst = gpu.construct_malloc_bdev(nb, bs, name="dbig2", device=0)
    try:
        gpu.bdev_write_raw(src, 1 << 30, traces.pattern_bytes(4, 0, 48 << 20))
        gpu.bdev_write_raw(src, size - 4096, traces.pattern_bytes(3, 0, 4096))
        gpu.bdev_image_track(src)
        gpu.bdev_image_save(src, tmp_path / "big.img")
        pieces = [(1 << 30, traces.pattern_bytes(5, 0, 48 << 20))]
        for g in rng.choice(nb, size=500, replace=False):
            pieces.append((int(g) * bs + int(rng.integers(0, bs - 64)), rng.integers(1, 256, size=64, dtype=np.uint8)))
        for off, data in pieces:
            gpu.bdev_write_raw(src, off, data)
        t0 = time.perf_counter()
        info = gpu.bdev_image_save_delta(src, tmp_path / "big.delta")
        t1 = time.perf_counter()
        granules = {off // GRANULE for off, _ in pieces[1:]}
        granules |= set(range((1 << 30) // GRANULE, ((1 << 30) + (48 << 20)) // GRANULE))
        assert info["data_bytes"] == GRANULE * len(granules) and info["zero_bytes"] == 0
        assert os.path.getsize(tmp_path / "big.delta") == info["file_bytes"]
        gpu.bdev_image_load(dst, tmp_path / "big.img")
        t2 = time.perf_counter()
        gpu.bdev_image_apply_delta(dst, tmp_path / "big.delta")
        t3 = time.perf_counter()
        assert gpu.bdev_digest(dst) == gpu.bdev_digest(src) == info["digest"]
        print(f"8 GiB, {info['data_bytes'] >> 20} MiB changed in {info['nextents']} runs: save_delta {t1 - t0:.3f} s, "
              f"load {t2 - t1:.3f} s, apply {t3 - t2:.3f} s")
    finally:
        gpu.delete_bdev(src)
        gpu.delete_bdev(dst)
