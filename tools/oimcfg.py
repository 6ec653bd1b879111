#!/usr/bin/env python
"""save / load the daemon's configuration over its JSON-RPC socket, the way SPDK's scripts/rpc.py save_config /
load_config do for the reference: `save` asks every subsystem for the calls that rebuild its state
(get_subsystems + get_subsystem_config, S/lib/event/rpc/subsystem_rpc.c:40-129) and prints
{"subsystems": [{"subsystem": ..., "config": [{"method", "params"}, ...]}, ...]}; `load` replays them in order.
  python tools/oimcfg.py save /var/tmp/spdk.sock > cfg.json
  python tools/oimcfg.py load /var/tmp/spdk.sock < cfg.json
With --images DIR, `save` also writes every bdev's bytes to DIR/<bdev>.img (save_bdev_image), and `load` fills each bdev
it constructs from DIR/<bdev>.img (load_bdev_image) before the vhost subsystem attaches anything to it:
  python tools/oimcfg.py save /var/tmp/spdk.sock --images /var/lib/oim/images > cfg.json
  python tools/oimcfg.py load /var/tmp/spdk.sock --images /var/lib/oim/images < cfg.json
An image file is never overwritten: save into an empty directory.
set_bdev_options is a start-up option of SPDK's bdev_io pools (no such pools here): it is saved for fidelity and
skipped on load."""
import json
import os
import socket
import sys


class Rpc:
    def __init__(self, path):
        self.s = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        self.s.connect(path)
        self.id = 0

    def call(self, method, params=None):
        self.id += 1
        req = {"jsonrpc": "2.0", "method": method, "id": self.id}
        if params is not None:
            req["params"] = params
        self.s.sendall((json.dumps(req) + "\n").encode())
        buf = b""
        while not buf.endswith(b"\n"):
            chunk = self.s.recv(1 << 20)
            if not chunk:
                raise ConnectionError("daemon closed the connection")
            buf += chunk
        rep = json.loads(buf)
        if "error" in rep:
            raise RuntimeError(f"{method}: code: {rep['error']['code']} msg: {rep['error']['message']}")
        return rep["result"]


def image_path(images: str, bdev: str) -> str:
    return os.path.join(os.path.abspath(images), bdev + ".img")


def save(rpc: Rpc, images: str | None = None) -> dict:
    cfg = {"subsystems": [{"subsystem": s["subsystem"], "config": rpc.call("get_subsystem_config", {"name": s["subsystem"]})}
                          for s in rpc.call("get_subsystems")]}
    if images is not None:
        for b in rpc.call("get_bdevs"):
            rpc.call("save_bdev_image", {"name": b["name"], "path": image_path(images, b["name"])})
    return cfg


def load(rpc: Rpc, cfg: dict, images: str | None = None) -> int:
    n = 0
    for sub in cfg["subsystems"]:
        made = []
        for item in sub["config"] or []:
            if item["method"] == "set_bdev_options":
                continue
            res = rpc.call(item["method"], item.get("params"))
            if sub["subsystem"] == "bdev" and item["method"].startswith("construct_"):
                made.append(res)        # the constructors answer with the bdev's name
            n += 1
        # the images go in before any later subsystem opens the bdevs
        for name in made if images is not None else []:
            rpc.call("load_bdev_image", {"name": name, "path": image_path(images, name)})
    return n


if __name__ == "__main__":
    args = sys.argv[1:]
    images = None
    if len(args) == 4 and args[2] == "--images":
        images = args[3]
        args = args[:2]
    if len(args) != 2 or args[0] not in ("save", "load"):
        sys.exit(__doc__)
    r = Rpc(args[1])
    if args[0] == "save":
        json.dump(save(r, images), sys.stdout, indent=2)
        print()
    else:
        print(f"{load(r, json.load(sys.stdin), images)} calls replayed", file=sys.stderr)
