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
With --track, `save` also enables image tracking on every bdev before its image is saved, so that later saves can write
only what changed: `save --deltas DIR` writes DIR/<bdev>.delta (save_bdev_image_delta), the granules each bdev changed
since its last image or delta, and `load --images DIR --deltas D1 D2 ...` applies each bdev's deltas in the order given
(apply_bdev_image_delta), after its image and before the vhost subsystem attaches anything to it:
  python tools/oimcfg.py save /var/tmp/spdk.sock --images /var/lib/oim/base --track > cfg.json
  python tools/oimcfg.py save /var/tmp/spdk.sock --deltas /var/lib/oim/d1 > /dev/null
  python tools/oimcfg.py load /var/tmp/spdk.sock --images /var/lib/oim/base --deltas /var/lib/oim/d1 < cfg.json
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


def image_path(images: str, bdev: str, ext: str = ".img") -> str:
    return os.path.join(os.path.abspath(images), bdev + ext)


def save(rpc: Rpc, images: str | None = None, track: bool = False, deltas: str | None = None) -> dict:
    cfg = {"subsystems": [{"subsystem": s["subsystem"], "config": rpc.call("get_subsystem_config", {"name": s["subsystem"]})}
                          for s in rpc.call("get_subsystems")]}
    for b in rpc.call("get_bdevs") if images is not None or deltas is not None else []:
        if deltas is not None:
            rpc.call("save_bdev_image_delta", {"name": b["name"], "path": image_path(deltas, b["name"], ".delta")})
        if images is not None:
            if track:
                rpc.call("enable_bdev_image_tracking", {"name": b["name"]})
            rpc.call("save_bdev_image", {"name": b["name"], "path": image_path(images, b["name"])})
    return cfg


def load(rpc: Rpc, cfg: dict, images: str | None = None, deltas: list[str] | tuple = ()) -> int:
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
            for d in deltas:
                rpc.call("apply_bdev_image_delta", {"name": name, "path": image_path(d, name, ".delta")})
    return n


def parse(args: list[str]):
    """-> (command, socket, images, track, deltas) or None: `save SOCK [--images DIR [--track]] [--deltas DIR]`,
    `load SOCK [--images DIR [--deltas DIR...]]`"""
    if len(args) < 2 or args[0] not in ("save", "load"):
        return None
    cmd, sock, rest = args[0], args[1], args[2:]
    images, track, deltas = None, False, []
    while rest:
        opt = rest.pop(0)
        if opt == "--images" and rest and images is None:
            images = rest.pop(0)
        elif opt == "--track" and cmd == "save" and not track:
            track = True
        elif opt == "--deltas" and rest and not deltas:
            while rest and not rest[0].startswith("--"):
                deltas.append(rest.pop(0))
        else:
            return None
    if (track and images is None) or (cmd == "save" and len(deltas) > 1) or (cmd == "load" and deltas and images is None):
        return None
    return cmd, sock, images, track, deltas


if __name__ == "__main__":
    p = parse(sys.argv[1:])
    if p is None:
        sys.exit(__doc__)
    cmd, sock, images, track, deltas = p
    r = Rpc(sock)
    if cmd == "save":
        json.dump(save(r, images, track, deltas[0] if deltas else None), sys.stdout, indent=2)
        print()
    else:
        print(f"{load(r, json.load(sys.stdin), images, deltas)} calls replayed", file=sys.stderr)
