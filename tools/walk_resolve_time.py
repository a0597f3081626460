"""regk_walk_resolve against regk_resolve on a watched walk kept current at 1 % churn.  The tree is
tools/walk_watch_time.py's fleet: S service records with I instances each (default 1 000 x 4 000).  After a complete
watched walk and a first (untimed) walk_resolve, one of two churns is applied, fed through the events, the refresh and
the new levels, and both resolves run on the same snapshot, alternated in one process (a warm-up, then best of five):
  (a) 1 % of instances deleted, 1 % created, 1 % of addresses changed, services untouched;
  (b) the same, plus every service rewritten with port 8080, so every SRV line and child run is fresh.
Each timed walk_resolve starts from the same kept text: the walk is rebuilt from the recorded streams before it.
Prints one JSON line per churn with kernel ms, copied / formatted bytes and segments, and the card's name and power
limit read in the same run.  --profile takes a per-kernel split of both calls with torch.profiler instead."""
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
import walk_watch_util as ww          # noqa: E402
from registrar_b200 import _native  # noqa: E402
from test_resolve_cpu import host, service  # noqa: E402

SESSION = 7
DH, DS = 30, 60


def dev(b):
    return torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()


def scenario(S, I, services_too):
    """-> (recorded walk levels, notifications, recorded refresh levels) of one churn"""
    rng = random.Random(1)
    zk = ww.WalkZooKeeper()
    zk.create(b"/fleet", b"", 0, False)
    for s in range(S):
        sp = b"/fleet/s%04d" % s
        zk.create(sp, service(b"_http", b"_tcp", 80, 60), 0, False)
        for i in range(I):
            zk.create(sp + b"/%07d" % i, host(b"redis_host", b"10.%d.%d.%d" % (s // 256, s % 256, i % 250), None, [6379]),
                      0, False)
    zk.take_events(SESSION)
    rec = []

    def recording(out):
        def exchange(fb):
            st = zk.serve(fb, SESSION)
            out.append((int(np.frombuffer(fb[4:8].tobytes(), ">i4")[0]), st))
            return st
        return exchange
    ctx = _native.Context(0)
    ctx.walk([b"/fleet"], recording(rec), watch=True)
    n = S * I // 100
    inst = [p for p in zk.nodes if p.count(b"/") == 3]
    picks = rng.sample(inst, 2 * n)
    for p in picks[:n]:
        zk.delete(p)
    for p in picks[n:]:
        zk.set_data(p, host(b"redis_host", b"10.250.%d.%d" % (rng.randrange(256), rng.randrange(250)), None, [6379]))
    for k in range(n):
        zk.create(b"/fleet/s%04d/n%07d" % (k % S, k), host(b"redis_host", b"10.200.%d.%d" % (k // 250 % 256, k % 250), None,
                                                          [6379]), 0, False)
    if services_too:
        for s in range(S):
            zk.set_data(b"/fleet/s%04d" % s, service(b"_http", b"_tcp", 8080, 60))
    notes = zk.take_events(SESSION)
    ctx.walk_events(np.frombuffer(notes, np.uint8))
    after = []
    ctx.refresh_walk(recording(after))
    ctx.close()
    return [(x, dev(s)) for x, s in rec], dev(notes), [(x, dev(s)) for x, s in after], n


def replay(ctx, before, notes, after):
    """the walk before the churn, a first walk_resolve, then the churn's events, refresh and levels"""
    ctx.walk_start([b"/fleet"])
    for x, s in before:
        ctx.walk_requests(x, device=True, watch=True)
        ctx.read_walk(s, device=True)
    ctx.walk_resolve(DH, DS, device=True)
    ctx.walk_events(notes, device=True)
    ctx.walk_refresh()
    for x, s in after:
        ctx.walk_requests(x, device=True, watch=True)
        w = ctx.read_walk(s, device=True)
    return w


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    profile = "--profile" in sys.argv
    S = int(args[0]) if args else 1000
    I = int(args[1]) if len(args) > 1 else 4000
    gpu = torch.cuda.get_device_name(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    for label, svc in (("a", False), ("b", True)):
        before, notes, after, n = scenario(S, I, svc)
        ctx, ctx2 = _native.Context(0), _native.Context(0)
        torch.cuda.synchronize()

        def incremental():
            replay(ctx, before, notes, after)
            out = ctx.walk_resolve(DH, DS, device=True)
            return dict(ms=float(out.answers.kernel_ms), launches=int(out.answers.launches),
                        copied=int(out.copied_bytes), formatted=int(out.formatted_bytes), n_fresh=int(out.n_fresh),
                        full=int(out.full), text=int(out.answers.text_total),
                        segments=int(ctx.get_option("walk_resolve_segments")))

        def plain():
            out = ctx2.resolve(ctx._walk, DH, DS, device=True)
            return dict(ms=float(out.kernel_ms), launches=int(out.launches), text=int(out.text_total))

        if profile:
            from torch.profiler import ProfilerActivity, profile as prof
            incremental(), plain()
            torch.cuda.synchronize()
            split = {}
            for name in ("walk_resolve", "resolve"):
                if name == "walk_resolve":
                    replay(ctx, before, notes, after)
                torch.cuda.synchronize()
                with prof(activities=[ProfilerActivity.CUDA]) as p:
                    if name == "walk_resolve":
                        ctx.walk_resolve(DH, DS, device=True)
                    else:
                        ctx2.resolve(ctx._walk, DH, DS, device=True)
                    torch.cuda.synchronize()
                rows = {}
                for e in p.key_averages():
                    t = getattr(e, "self_device_time_total", None)
                    t = e.self_cuda_time_total if t is None else t
                    if t:
                        rows[e.key[:60]] = round(t / 1000.0, 3)
                split[name] = dict(sorted(rows.items(), key=lambda kv: -kv[1]))
            print(json.dumps({"churn": label, "workload": "fleet %d x %d" % (S, I), "profile_ms": split, "gpu": gpu,
                              "power_limit_max_sm_clock": card}), flush=True)
        else:
            incremental(), plain()                                  # warm-up
            inc, ful = [], []
            for _ in range(5):
                inc.append(incremental())
                ful.append(plain())
            bi = min(inc, key=lambda r: r["ms"])
            bf = min(ful, key=lambda r: r["ms"])
            assert bi["text"] == bf["text"] and bi["full"] == 0
            print(json.dumps({
                "churn": label, "workload": "fleet %d x %d, 1%% deleted / created / readdressed%s" % (
                    S, I, ", every service rewritten" if svc else ""), "churn_nodes": n,
                "best_walk_resolve_ms": round(bi["ms"], 3), "best_resolve_ms": round(bf["ms"], 3),
                "speedup": round(bf["ms"] / bi["ms"], 2) if bi["ms"] else None,
                "walk_resolve_launches": bi["launches"], "resolve_launches": bf["launches"],
                "text_total": bi["text"], "copied_bytes": bi["copied"], "formatted_bytes": bi["formatted"],
                "n_fresh": bi["n_fresh"], "segments": bi["segments"],
                "gpu": gpu, "power_limit_max_sm_clock": card}), flush=True)
        ctx.close()
        ctx2.close()


if __name__ == "__main__":
    main()
