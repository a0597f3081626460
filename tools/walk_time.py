"""The registry walk on the fleet tree of tools/resolve_time.py: 4 M config 2 records collapsed onto 1 000 domains, one
service record per domain directory.  The walk starts at the 1 000 service directories: level 0 reads the service records
and lists their instances, level 1 reads the 4 M instances (and lists their empty child sets).  Each level's reply stream
(getData replies, then getChildren replies) is built on the device before the timed window.  After a warm-up walk, five
walks are timed; each is followed by regk_resolve on the walk's snapshot, and resolve runs once more on its own on that
snapshot.  Prints one JSON line: per level kernel ms (framing + read), launches, request and reply bytes; the whole walk,
walk + resolve and resolve alone (best of five), and the card's name and power limit read in the same run."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import replies_util as ru    # noqa: E402
import walk_util as wu       # noqa: E402
from registrar_b200 import _native  # noqa: E402
from resolve_time import SERVICE, fleet  # noqa: E402


def be(v, w):
    return np.ascontiguousarray(np.asarray(v).astype(">i%d" % w)).view(np.uint8).reshape(-1, w)


def gather(bytes_, off, order, chunk=1 << 19):
    """the strings bytes_[off[i]:off[i+1]] for i in order, packed on the device in chunks: (host bytes, offsets)"""
    lens = (off[1:] - off[:-1])[order]
    no = np.zeros(len(order) + 1, np.int64)
    np.cumsum(lens, out=no[1:])
    src, out = torch.from_numpy(bytes_).cuda(), torch.empty(int(no[-1]), dtype=torch.uint8, device="cuda")
    for a in range(0, len(order), chunk):
        b = min(len(order), a + chunk)
        ln = torch.from_numpy(lens[a:b]).cuda()
        start = torch.from_numpy(off[:-1][order[a:b]]).cuda()
        rep = torch.repeat_interleave(torch.arange(b - a, device="cuda"), ln)
        within = torch.arange(rep.numel(), device="cuda") - (torch.cumsum(ln, 0) - ln)[rep]
        out[int(no[a]):int(no[b])] = src[start[rep] + within]
    return out.cpu().numpy(), no


def streams(res, idx, ndom):
    """roots, and each level's reply stream as a CUDA tensor"""
    po, jo = res.path_off.astype(np.int64), res.json_off.astype(np.int64)
    pb, jb = res.path_bytes, res.json_bytes
    _, first = np.unique(idx, return_index=True)
    roots = []
    for i in first.tolist():
        p = pb[po[i]:po[i + 1]].tobytes()
        roots.append(p[:p.rfind(b"/")])
    assert wu.root_error(roots) is None and len(roots) == ndom
    order = np.argsort(idx, kind="stable")                  # level 1: each directory's instances, in record order
    dlen = np.array([len(r) for r in roots], np.int64)[idx[order]]
    # level 0: the service records, then each directory's listing (its instances' names)
    f0 = len(roots)
    gd0 = b"".join(ru.success(1 + k, SERVICE, seed=k) for k in range(f0))
    name_off = po[:-1][order] + dlen + 1
    name_len = po[1:][order] - name_off
    ent_len = 4 + name_len
    eo = np.zeros(len(order) + 1, np.int64)
    np.cumsum(ent_len, out=eo[1:])
    ent = np.zeros(int(eo[-1]), np.uint8)
    ent[(eo[:-1][:, None] + np.arange(4)[None, :]).reshape(-1)] = be(name_len, 4).reshape(-1)
    within = np.arange(int(name_len.sum())) - np.repeat(np.cumsum(name_len) - name_len, name_len)
    ent[np.repeat(eo[:-1] + 4, name_len) + within] = pb[np.repeat(name_off, name_len) + within]
    cnt = np.bincount(idx, minlength=ndom)
    co = np.concatenate([[0], np.cumsum(cnt)])
    gc0 = []
    for k in range(f0):
        e = ent[eo[co[k]]:eo[co[k + 1]]].tobytes()
        hdr = np.array([20 + len(e)], ">i4").tobytes() + np.array([1 + f0 + k], ">i4").tobytes() + bytes(8) + bytes(4) + \
            np.array([cnt[k]], ">i4").tobytes()
        gc0.append(hdr + e)
    s0 = torch.from_numpy(np.frombuffer(gd0 + b"".join(gc0), np.uint8).copy()).cuda()
    # level 1: the instances' getData replies (built on the device), then their empty listings
    n = len(order)
    x1 = 1 + 2 * f0
    jbo, joo = gather(jb, jo, order)
    gd1 = ru.device_replies(jbo, joo.astype(np.uint64), x1, np.arange(n, dtype=np.int32) % 7, np.full(n, 0x55, np.int64))
    h = np.zeros((n, 24), np.uint8)
    h[:, 0:4] = be(np.full(n, 20), 4)
    h[:, 4:8] = be((x1 + n + np.arange(n, dtype=np.int64) + 2 ** 31) % 2 ** 32 - 2 ** 31, 4)
    gc1 = torch.from_numpy(h.reshape(-1)).cuda()
    s1 = torch.cat([gd1, gc1])
    return roots, [(1, s0), (x1, s1)]


def walk_once(ctx, roots, levels):
    ctx.walk_start(roots)
    rows, w = [], None
    t0 = time.perf_counter()
    for xid, s in levels:
        fr = ctx.walk_requests(xid, device=True)
        w = ctx.read_walk(s, device=True)
        rows.append(dict(frame_ms=float(fr.kernel_ms), read_ms=float(w.kernel_ms), launches=1 + int(w.launches),
                         request_bytes=int(fr.total), reply_bytes=s.numel(), nodes=int(w.n_found),
                         children=int(w.n_children)))
    wall = (time.perf_counter() - t0) * 1e3
    assert int(w.n_frontier) == 0 and rows[0]["children"] == rows[1]["nodes"] and int(w.n_error) == 0
    return rows, wall, w


def main():
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    b, idx = fleet(int(4_000_000 * scale))
    res = ctx.register_batch(b)
    roots, levels = streams(res, idx, 1000)
    del res
    torch.cuda.synchronize()
    walk_once(ctx, roots, levels)                           # warm-up
    runs = []
    for _ in range(5):
        rows, wall, w = walk_once(ctx, roots, levels)
        wobj = _native.Walk(ctx, w)
        a = ctx.resolve(wobj, 30, 60, device=True)
        a2 = ctx.resolve(wobj, 30, 60, device=True)         # resolve alone, on the same snapshot
        runs.append((rows, wall, float(a.kernel_ms), float(a2.kernel_ms), int(w.m), int(a.text_total)))
    best = min(runs, key=lambda r: sum(x["frame_ms"] + x["read_ms"] for x in r[0]))
    walk_ms = [sum(x["frame_ms"] + x["read_ms"] for x in r[0]) for r in runs]
    print(json.dumps({
        "workload": "fleet walk", "records": len(idx), "services": len(roots), "m": best[4], "levels": best[0],
        "walk_kernel_ms": [round(v, 3) for v in walk_ms], "best_walk_kernel_ms": round(min(walk_ms), 3),
        "best_walk_wall_ms": round(min(r[1] for r in runs), 3),
        "best_walk_plus_resolve_ms": round(min(wm + r[2] for wm, r in zip(walk_ms, runs)), 3),
        "best_resolve_alone_ms": round(min(r[3] for r in runs), 3), "text_bytes": best[5],
        "gpu": gpu, "power_limit_max_sm_clock": power}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
