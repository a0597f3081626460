"""The watched round against the full stat round on 10 M config 3 records (EVENTS_N overrides), one registry state for
both: 1 % of the nodes fired (half NodeDataChanged, half NodeDeleted) and about 1 k service
directories fired NodeChildrenChanged.  Streams are built on the host once and staged on the device.  Measured:
  first     the first regk_read_events after the batch finished (one sample; its buffers grow inside the timed span, and
            the table build it starts with runs before that span)
  events    a steady-state regk_read_events of the same stream
  requests  regk_events_requests(REGK_ZK_EXISTS) + (REGK_ZK_GETCHILDREN), wall clock (host steps included)
  subset    regk_read_stats + regk_reconcile_stats over the dirty records' replies
  full      the full stat round: regk_jute_requests(REGK_ZK_EXISTS) framed, regk_read_stats + regk_reconcile_stats
The watched and the full round alternate five times after a warm-up of each.  Kernel ms are the library's own events.
One JSON line per measurement, with the card's name and power limit read in the same run."""
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
from registrar_b200 import _native, synth
import children_util as cu
import events_util as eu
from test_read_stats import device_stat_replies

N = int(os.environ.get("EVENTS_N", 10_000_000))
SESSION = 0x1234_5678_9ABC_DEF0


def main():
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    card = {"gpu": gpu, "power_limit_max_sm_clock": power}
    ctx = _native.Context(0)
    res = ctx.register_batch(synth.generate("config3", n=N))
    n = res.n
    rng = np.random.default_rng(7)
    fired = np.sort(rng.permutation(n)[:n // 100])
    deleted = fired[::2]
    po = res.path_off.astype(np.int64)
    pb = res.path_bytes
    path = lambda i: pb[po[i]:po[i + 1]].tobytes()
    paths_small = [path(i) for i in range(min(n, 200_000))]
    dirs = [d for _, d in cu.dir_set(paths_small)[0]][:1000]
    dset = set(deleted.tolist())
    parts = [eu.notification(path(i), eu.DELETED if i in dset else eu.DATA_CHANGED) for i in fired.tolist()]
    parts += [eu.notification(d, eu.CHILDREN_CHANGED) for d in dirs]
    stream = torch.from_numpy(np.frombuffer(b"".join(parts), np.uint8).copy()).cuda()
    jo = res.json_off.astype(np.int64)
    dlen_all = np.diff(jo).astype(np.int32)
    missing = np.zeros(n, bool)
    missing[deleted] = True
    dl = dlen_all.copy()
    dl[fired] += 1
    s_full, _ = device_stat_replies(n, 1, np.ones(n, np.int32), np.full(n, SESSION, np.int64), dl, np.ones(n, np.int64),
                                    missing)
    del res, pb
    torch.cuda.synchronize()
    first = float(ctx.read_events(stream, device=True).kernel_ms)      # the tables are built here
    ev = ctx.read_events(stream, device=True)
    m = int(ev.n_dirty_recs)                                            # DUP paths map to their first record
    # the replies to the subset re-check: every dirty node found at another data length
    s_sub, _ = device_stat_replies(m, 1, np.ones(m, np.int32), np.full(m, SESSION, np.int64), np.full(m, 1, np.int32),
                                   np.ones(m, np.int64), np.zeros(m, bool))
    torch.cuda.synchronize()

    def watched_round():
        ev = ctx.read_events(stream, device=True)
        assert int(ev.n_dirty_recs) == m and int(ev.n_dirty_dirs) == len(dirs)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fe = ctx.events_requests(_native.ZK_EXISTS, xid_base=1, device=True)
        fc = ctx.events_requests(_native.ZK_GETCHILDREN, xid_base=1 + m, device=True)
        req_ms = (time.perf_counter() - t0) * 1e3
        st = ctx.read_stats(s_sub, device=True)
        d = ctx.reconcile_stats(st, session=SESSION, zk_flags=1, device=True)
        assert int(d.d.n_update) + int(d.d.n_same) + int(d.d.n_dup) == n
        return {"events_ms": float(ev.kernel_ms), "requests_wall_ms": req_ms, "read_ms": float(st.kernel_ms),
                "reconcile_ms": float(d.d.kernel_ms), "request_bytes": int(fe.total) + int(fc.total)}

    def full_round():
        fr = ctx.jute_requests(_native.ZK_EXISTS, xid_base=1, device=True)
        st = ctx.read_stats(s_full, device=True)
        d = ctx.reconcile_stats(st, session=SESSION, zk_flags=1, device=True)
        assert int(d.d.n_create) > 0
        return {"read_ms": float(st.kernel_ms), "reconcile_ms": float(d.d.kernel_ms), "request_bytes": int(fr.total)}

    watched_round(), full_round()
    rows = {"watched": [], "full": []}
    for _ in range(5):
        rows["watched"].append(watched_round())
        rows["full"].append(full_round())
    w, f = rows["watched"], rows["full"]
    print(json.dumps(dict(card, round="watched", n=n, fired_records=m, fired_dirs=len(dirs),
                          first_read_events_kernel_ms=round(first, 3),
                          read_events_kernel_ms=[round(x["events_ms"], 3) for x in w],
                          events_requests_wall_ms=[round(x["requests_wall_ms"], 3) for x in w],
                          subset_stats_kernel_ms=[round(x["read_ms"] + x["reconcile_ms"], 3) for x in w],
                          best_read_events_ms=min(round(x["events_ms"], 3) for x in w),
                          best_subset_stats_ms=min(round(x["read_ms"] + x["reconcile_ms"], 3) for x in w),
                          event_stream_bytes=stream.numel(), request_bytes=w[0]["request_bytes"],
                          reply_bytes=s_sub.numel())), flush=True)
    print(json.dumps(dict(card, round="full", n=n,
                          stats_kernel_ms=[round(x["read_ms"] + x["reconcile_ms"], 3) for x in f],
                          best_stats_kernel_ms=min(round(x["read_ms"] + x["reconcile_ms"], 3) for x in f),
                          request_bytes=f[0]["request_bytes"], reply_bytes=s_full.numel())), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
