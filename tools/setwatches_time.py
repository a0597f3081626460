"""Re-arming a watched registry after a reconnect: SetWatches against round 0, on 10 M config 3 records (SETWATCHES_N
overrides), every record and service directory armed, 1 % of the records changed while the connection was down.
Streams are built on the host once and staged on the device.  Measured:
  setwatches  regk_setwatches_requests: kernel ms (the library's events), wall ms (host steps included), frame bytes
  events      regk_read_events over the server's answer: the notifications of what changed and the SetWatches replies
  subset      the re-check: regk_events_requests(REGK_ZK_EXISTS) wall ms, regk_read_stats + regk_reconcile_stats kernel ms
  round0      the same registry re-armed by round 0: exists and getChildren framed with the watch byte and read back
              (regk_read_stats + regk_read_children kernel ms, and the wall ms of the four calls)
The two routes alternate five times after a warm-up of each.  One JSON line per route, with the card's name and power
limit read in the same run."""
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
import events_util as eu
import setwatches_util as sw
import stats_util as su
from test_read_stats import device_stat_replies

N = int(os.environ.get("SETWATCHES_N", 10_000_000))
SESSION = 0x1234_5678_9ABC_DEF0
DIR_XID = 1 << 30


def children_replies(d, xid_base, zxid):
    """an empty listing for each of d directories: len 20 | xid | zxid | err 0 | count 0"""
    fr = np.zeros(d, np.dtype([("len", ">i4"), ("xid", ">i4"), ("zxid", ">i8"), ("err", ">i4"), ("cnt", ">i4")]))
    fr["len"] = 20
    fr["xid"] = ((xid_base + np.arange(d, dtype=np.int64) + 2 ** 31) % 2 ** 32 - 2 ** 31).astype(np.int32)
    fr["zxid"] = zxid
    return torch.from_numpy(fr.view(np.uint8).copy()).cuda()


def main():
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    card = {"gpu": gpu, "power_limit_max_sm_clock": power}
    ctx = _native.Context(0)
    res = ctx.register_batch(synth.generate("config3", n=N))
    n = res.n
    dlen = np.diff(res.json_off.astype(np.int64)).astype(np.int32)
    po, pb = res.path_off.astype(np.int64), res.path_bytes
    path = lambda i: pb[po[i]:po[i + 1]].tobytes()
    s_full, _ = device_stat_replies(n, 1, np.zeros(n, np.int32), np.full(n, SESSION, np.int64), dlen,
                                    np.ones(n, np.int64), np.zeros(n, bool))
    fc = ctx.children_requests(_native.ZK_GETCHILDREN, xid_base=DIR_XID, watch=True, device=True)
    d = int(fc.n)
    s_dirs = children_replies(d, DIR_XID, 100)
    rng = np.random.default_rng(7)
    changed = np.sort(rng.permutation(n)[:n // 100])

    def round0():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fe = ctx.jute_requests(_native.ZK_EXISTS, xid_base=1, watch=True, device=True)
        st = ctx.read_stats(s_full, device=True)
        fc = ctx.children_requests(_native.ZK_GETCHILDREN, xid_base=DIR_XID, watch=True, device=True)
        ch = ctx.read_children(s_dirs, device=True)
        wall = (time.perf_counter() - t0) * 1e3
        return {"kernel_ms": float(st.kernel_ms) + float(ch.kernel_ms), "wall_ms": wall,
                "request_bytes": int(fe.total) + int(fc.total), "reply_bytes": s_full.numel() + s_dirs.numel()}

    round0()
    sg = ctx.setwatches_requests()
    assert sg.n_data > 0 and sg.n_repend_recs == 0 and sg.n_repend_dirs == 0
    # the server's answer: NodeDataChanged for every changed record, then one reply per frame
    parts = [eu.notification(path(i), eu.DATA_CHANGED) for i in changed.tolist()]
    answer = torch.from_numpy(np.frombuffer(b"".join(parts) + sw.reply(100) * sg.n_frames, np.uint8).copy()).cuda()
    ev = ctx.read_events(answer, device=True)
    m = int(ev.n_dirty_recs)
    s_sub, _ = device_stat_replies(m, 1, np.ones(m, np.int32), np.full(m, SESSION, np.int64), np.full(m, 1, np.int32),
                                   np.ones(m, np.int64), np.zeros(m, bool))
    ctx.events_requests(_native.ZK_EXISTS, xid_base=1, device=True)
    ctx.read_stats(s_sub, device=True)
    del res, pb

    def reconnect():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sg = ctx.setwatches_requests(device=True)
        sw_wall = (time.perf_counter() - t0) * 1e3
        ev = ctx.read_events(answer, device=True)
        assert int(ev.n_dirty_recs) == m and int(ev.n_replies) == int(sg.frames.n)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fe = ctx.events_requests(_native.ZK_EXISTS, xid_base=1, device=True)
        req_wall = (time.perf_counter() - t0) * 1e3
        st = ctx.read_stats(s_sub, device=True)
        dd = ctx.reconcile_stats(st, session=SESSION, zk_flags=1, device=True)
        return {"setwatches_kernel_ms": float(sg.frames.kernel_ms), "setwatches_wall_ms": sw_wall,
                "frame_bytes": int(sg.frames.total), "frames": int(sg.frames.n), "listed": int(sg.n_data + sg.n_exist +
                sg.n_child), "read_events_kernel_ms": float(ev.kernel_ms), "requests_wall_ms": req_wall,
                "subset_kernel_ms": float(st.kernel_ms) + float(dd.d.kernel_ms), "request_bytes": int(fe.total)}

    reconnect(), round0()
    rows = {"setwatches": [], "round0": []}
    for _ in range(5):
        rows["setwatches"].append(reconnect())
        rows["round0"].append(round0())
    w, r = rows["setwatches"], rows["round0"]
    best = lambda rows, k: min(round(x[k], 3) for x in rows)
    print(json.dumps(dict(card, route="setwatches", n=n, dirs=d, changed=m, frames=w[0]["frames"],
                          listed=w[0]["listed"], frame_bytes=w[0]["frame_bytes"], answer_bytes=answer.numel(),
                          recheck_request_bytes=w[0]["request_bytes"], recheck_reply_bytes=s_sub.numel(),
                          best_setwatches_kernel_ms=best(w, "setwatches_kernel_ms"),
                          best_setwatches_wall_ms=best(w, "setwatches_wall_ms"),
                          best_read_events_kernel_ms=best(w, "read_events_kernel_ms"),
                          best_events_requests_wall_ms=best(w, "requests_wall_ms"),
                          best_subset_kernel_ms=best(w, "subset_kernel_ms"),
                          setwatches_kernel_ms=[round(x["setwatches_kernel_ms"], 3) for x in w])), flush=True)
    print(json.dumps(dict(card, route="round0", n=n, dirs=d, request_bytes=r[0]["request_bytes"],
                          reply_bytes=r[0]["reply_bytes"], best_kernel_ms=best(r, "kernel_ms"),
                          best_wall_ms=best(r, "wall_ms"), kernel_ms=[round(x["kernel_ms"], 3) for x in r])), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
