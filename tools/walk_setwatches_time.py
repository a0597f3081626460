"""A watched walk carried across a reconnect at 1 % churn, against a full re-walk of the same tree state.  The tree and
the churn are tools/walk_watch_time.py's: a fleet of S service records with I instances each (default 1 000 x 1 000),
walked with watches; then the connection drops, and while it is down half of 1 % of the instances are deleted, as many
are created, and every service record's data is rewritten.  The tree is served by
tests/walk_setwatches_util.TreeZooKeeper, which answers SetWatches as DataTree.setWatches does.  Every stream is
recorded once through the server and replayed from device memory, so the timed rounds measure the library alone.  Each
round (a warm-up, then five) runs on one context: the watched walk before the churn (not timed), regk_walk_setwatches,
the SetWatches replies and the notifications they fire (regk_walk_events), regk_walk_refresh and the levels it reads;
then a full walk of the tree after the churn on a second context, alternated in the same process.  Prints one JSON line
with the best of five, the bytes each way, and the card's name, power limit and max SM clock read in the same run."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import walk_setwatches_util as ws   # noqa: E402
from registrar_b200 import _native  # noqa: E402
from test_resolve_cpu import host, service  # noqa: E402

SESSION = 7


def record(zk, roots, ctx, watch):
    """a walk through the tree server, every level's (xid, stream) kept; the walk runs on ctx"""
    out = []

    def exchange(fb):
        s = zk.serve(fb, SESSION)
        out.append((int(np.frombuffer(fb[4:8].tobytes(), ">i4")[0]), s))
        return s
    ctx.walk(roots, exchange, watch=watch)
    return out


def dev(b):
    return torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()


def main():
    S = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
    I = int(sys.argv[2]) if len(sys.argv) > 2 else 1000
    rng = random.Random(1)
    gpu = torch.cuda.get_device_name(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    zk = ws.TreeZooKeeper()
    zk.create(b"/fleet", b"", 0, False)
    for s in range(S):
        sp = b"/fleet/s%04d" % s
        zk.create(sp, service(b"_http", b"_tcp", 80, 60), 0, False)
        for i in range(I):
            zk.create(sp + b"/%07d" % i, host(b"redis_host", b"10.%d.%d.%d" % (s // 256, s % 256, i % 250), None, [6379]),
                      0, False)
    zk.take_events(SESSION)
    ctx, ctx2 = _native.Context(0), _native.Context(0)
    before = record(zk, [b"/fleet"], ctx, True)
    zk.drop_connection(SESSION)
    n_churn = S * I // 200
    inst = [p for p in zk.nodes if p.count(b"/") == 3]
    for p in rng.sample(inst, n_churn):
        zk.delete(p)
    for k in range(n_churn):
        zk.create(b"/fleet/s%04d/n%07d" % (k % S, k), host(b"redis_host", b"10.200.%d.%d" % (k // 250 % 256, k % 250), None,
                                                          [6379]), 0, False)
    for s in range(S):
        zk.set_data(b"/fleet/s%04d" % s, service(b"_http", b"_tcp", 8080, 60))
    sw = ctx.walk_setwatches()
    sw_frames = sw.frames.tobytes()
    sw_stream = zk.serve_setwatches(sw_frames, SESSION)
    e0 = ctx.walk_events(np.frombuffer(sw_stream, np.uint8))
    after_levels = []

    def exchange(fb):
        s = zk.serve(fb, SESSION)
        after_levels.append((int(np.frombuffer(fb[4:8].tobytes(), ">i4")[0]), s))
        return s
    r0, w0 = ctx.refresh_walk(exchange)
    full = record(zk, [b"/fleet"], ctx2, False)
    d_before = [(x, dev(s)) for x, s in before]
    d_after = [(x, dev(s)) for x, s in after_levels]
    d_full = [(x, dev(s)) for x, s in full]
    d_sw = dev(sw_stream)
    torch.cuda.synchronize()

    def resume_round():
        ctx.walk_start([b"/fleet"])
        for x, s in d_before:
            ctx.walk_requests(x, device=True, watch=True)
            ctx.read_walk(s, device=True)
        fr = ctx.walk_setwatches(device=True)
        e = ctx.walk_events(d_sw, device=True)
        r = ctx.walk_refresh()
        row = dict(setwatches_ms=float(fr.frames.kernel_ms), setwatches_bytes=int(fr.frames.total),
                   n_listed=int(fr.n_listed), events_ms=float(e.kernel_ms), table_ms=float(e.table_ms),
                   n_events=int(e.n_events), refresh_ms=float(r.kernel_ms), n_removed=r.n_removed,
                   n_frontier=r.n_frontier, levels_ms=0.0, request_bytes=0, reply_bytes=0)
        for x, s in d_after:
            q = ctx.walk_requests(x, device=True, watch=True)
            w = ctx.read_walk(s, device=True)
            row["levels_ms"] += float(q.kernel_ms) + float(w.kernel_ms)
            row["request_bytes"] += int(q.total)
            row["reply_bytes"] += s.numel()
        return row

    def full_round():
        ctx2.walk_start([b"/fleet"])
        ms, req, rep = 0.0, 0, 0
        for x, s in d_full:
            fr = ctx2.walk_requests(x, device=True)
            w = ctx2.read_walk(s, device=True)
            ms += float(fr.kernel_ms) + float(w.kernel_ms)
            req, rep = req + int(fr.total), rep + s.numel()
        return dict(ms=ms, request_bytes=req, reply_bytes=rep, m=int(w.m))

    resume_round(), full_round()                           # warm-up
    rows, fulls = [], []
    for _ in range(5):
        rows.append(resume_round())
        fulls.append(full_round())
    best = lambda k: round(min(r[k] for r in rows), 3)    # noqa: E731
    row = rows[0]
    resume_wire = row["setwatches_bytes"] + len(sw_stream) + row["request_bytes"] + row["reply_bytes"]
    full_wire = fulls[0]["request_bytes"] + fulls[0]["reply_bytes"]
    print(json.dumps({
        "workload": "fleet %d x %d, 1%% churn while the connection is down" % (S, I), "deleted": n_churn,
        "created": n_churn, "services_rewritten": S, "snapshot_nodes": int(w0.m),
        "n_listed": row["n_listed"], "setwatches_frames": int(sw.n_frames), "setwatches_bytes": row["setwatches_bytes"],
        "best_setwatches_ms": best("setwatches_ms"),
        "setwatches_reply_stream_bytes": len(sw_stream), "notifications_fired": int(e0.n_events),
        "best_events_ms": best("events_ms"), "best_table_ms": best("table_ms"),
        "refresh_removed": row["n_removed"], "refresh_frontier": row["n_frontier"], "best_refresh_ms": best("refresh_ms"),
        "best_refresh_levels_ms": best("levels_ms"), "refresh_request_bytes": row["request_bytes"],
        "refresh_reply_bytes": row["reply_bytes"], "resume_wire_bytes": resume_wire,
        "best_resume_kernel_ms": round(min(r["setwatches_ms"] + r["events_ms"] + r["table_ms"] + r["refresh_ms"] +
                                           r["levels_ms"] for r in rows), 3),
        "best_full_walk_ms": round(min(f["ms"] for f in fulls), 3), "full_walk_request_bytes": fulls[0]["request_bytes"],
        "full_walk_reply_bytes": fulls[0]["reply_bytes"], "full_walk_wire_bytes": full_wire, "full_walk_m": fulls[0]["m"],
        "same_node_count_as_full_walk": int(w0.m) == fulls[0]["m"],
        "gpu": gpu, "power_limit_max_sm_clock": card}), flush=True)
    ctx.close()
    ctx2.close()


if __name__ == "__main__":
    main()
