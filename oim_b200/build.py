"""Build liboimgpu.so (hand-written sm_90a kernels + the C-ABI host side) in-tree with nvcc.

nvcc cross-compiles without a GPU; the resulting .so is a build product and stays out of git.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "liboimgpu.so")
SOURCES = ["control.cu", "session.cu", "nbd.cu", "copy_chan.cu", "bio_chan.cu", "mirror_check.cu", "bdev_image.cu", "image_delta.cu",
           "lun_kernel.cu"]
HEADERS = ["host_state.h", "bdev_image.h", "lun_kernel.cuh", os.path.join(ROOT, "include", "oimgpu.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC,-Wall", "-shared", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, defs: str | None = None, out: str = LIB) -> str:
    """defs: extra -D flags for tuning builds (e.g. "-DOIM_MOVERS=8 -DOIM_MIN_BLOCKS=2")."""
    defs = defs if defs is not None else os.environ.get("OIM_NVCC_DEFS", "")
    if os.environ.get("OIM_LIB_PATH") and out == LIB:
        return os.environ["OIM_LIB_PATH"]           # a tuning build was selected explicitly
    if not force and not defs and out == LIB and not _stale():
        build_daemon()
        return LIB
    cmd = [NVCC, *FLAGS, *defs.split(), "-Xptxas", "-v", "-o", out, *[os.path.join(CSRC, s) for s in SOURCES]]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout[-4000:] + res.stderr[-4000:])
    if verbose:
        print(res.stderr[-3000:])
    if out == LIB:
        build_daemon()
    return out


DAEMON = os.path.join(HERE, "oim-gpu-vhost")
DAEMON_SRC = os.path.join(HERE, "daemon", "oim_gpu_vhost.cpp")
DAEMON_SRCS = [DAEMON_SRC, os.path.join(HERE, "daemon", "vhost_user.cpp")]
DAEMON_DEPS = DAEMON_SRCS + [os.path.join(HERE, "daemon", "vhost_user.h")]


def build_daemon(force: bool = False) -> str:
    """the JSON-RPC daemon (drop-in for SPDK's `vhost` binary): plain C++ on top of the C ABI"""
    if not force and os.path.exists(DAEMON) and os.path.getmtime(DAEMON) >= max(
            *[os.path.getmtime(d) for d in DAEMON_DEPS], os.path.getmtime(LIB), os.path.getmtime(os.path.join(ROOT, "include", "oimgpu.h"))):
        return DAEMON
    cmd = ["g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-rdynamic", "-g", "-I", os.path.join(ROOT, "include"), "-o", DAEMON, *DAEMON_SRCS,
           "-L", HERE, "-loimgpu", "-Wl,-rpath,$ORIGIN"]
    out = subprocess.run(cmd, capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("daemon build failed:\n" + out.stdout[-3000:] + out.stderr[-3000:])
    return DAEMON


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print(LIB)
