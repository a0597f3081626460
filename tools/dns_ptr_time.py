"""regk_dns_answer with and without REGK_DNS_PTR on the fleet of tools/dns_time.py (4 M config 2 records collapsed onto
1 000 domains plus one service record per domain, device snapshot).  The query mix is dns_time's with a PTR share: 80 %
of dns_time's UDP mix and 20 % PTR queries for the reverse names of 50 000 sampled records' addresses (a tenth of them
for absent addresses).  The same device-resident messages are answered with and without the flag, alternated in one
process: one warm-up each, then five rounds (best kernel_ms of each).  The once-per-resolve reverse index is timed on
its own: the first one-message PTR call after a resolve minus the same call again (the preparation pass, which a
flag-less call would also run, is taken out by a flag-less call first).  Prints one JSON line per measurement with the
card's name and power limit read in the same run."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from registrar_b200 import _native
from resolve_time import fleet, snapshot
from dns_time import queries
import dns_ptr_util as pu
import dns_util as du


def ptr_queries(res, k, rng):
    """k device-resident PTR messages over sampled records' addresses"""
    jo = res.json_off.astype(np.int64)
    pool = []
    for i in rng.choice(res.n, 50_000, replace=False).tolist():
        d = res.json_bytes[jo[i]:jo[i + 1]].tobytes()
        s = d.find(b'"address":"') + 11
        pool.append(du.query(pu.reverse_name(d[s:d.index(b'"', s)]), pu.T_PTR))
    pool += [du.query(pu.reverse_name(b"192.168.%d.%d" % (j // 250, j % 250 + 1)), pu.T_PTR) for j in range(5000)]
    pick = rng.integers(0, len(pool), k)
    lens = np.array([len(x) for x in pool], np.int64)
    starts = np.zeros(len(pool), np.int64)
    np.cumsum(lens[:-1], out=starts[1:])
    off = np.zeros(k + 1, np.int64)
    np.cumsum(lens[pick], out=off[1:])
    blob = torch.from_numpy(np.frombuffer(b"".join(pool), np.uint8).copy()).cuda()
    doff, dpick, dstart = torch.from_numpy(off).cuda(), torch.from_numpy(pick).cuda(), torch.from_numpy(starts).cuda()
    pos = torch.arange(int(off[-1]), device="cuda", dtype=torch.int64)
    which = torch.searchsorted(doff[1:], pos, right=True)
    return blob[dstart[dpick[which]] + pos - doff[which]], doff


def mix(res, idx, k, rng):
    """dns_time's messages, then the PTR messages"""
    fwd, foff = queries(res, idx, k - k // 5, rng)
    ptr, poff = ptr_queries(res, k // 5, rng)
    return torch.cat([fwd, ptr]), torch.cat([foff, foff[-1] + poff[1:]])


def main():
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    b, idx = fleet(int(4_000_000 * scale))
    res = ctx.register_batch(b)
    snap = snapshot(res, idx)
    one_m, one_o = du.pack([du.query(b"1.0.0.10.in-addr.arpa", pu.T_PTR)])
    builds = []
    for _ in range(5):
        ctx.resolve(snap, 30, 60, device=True)
        ctx.answer_dns(one_m, one_o, device=True)
        first = ctx.answer_dns(one_m, one_o, device=True, ptr=True)
        again = ctx.answer_dns(one_m, one_o, device=True, ptr=True)
        builds.append(float(first.kernel_ms) - float(again.kernel_ms))
    print(json.dumps({"index_build_ms": [round(x, 3) for x in builds], "best_index_build_ms": round(min(builds), 3),
                      "m": snap.m, "launches_first_ptr_call": int(first.launches), "launches_after": int(again.launches),
                      "gpu": gpu, "power_limit_max_sm_clock": power}), flush=True)
    rng = np.random.default_rng(7)
    k = int(10_000_000 * scale)
    msgs, off = mix(res, idx, k, rng)
    ms = {False: [], True: []}
    outs = {}
    for flag in (False, True):
        ctx.answer_dns(msgs, off, 1232, device=True, ptr=flag)
    for _ in range(5):
        for flag in (False, True):
            out = ctx.answer_dns(msgs, off, 1232, device=True, ptr=flag)
            ms[flag].append(float(out.kernel_ms))
            outs[flag] = (list(out.n_status), int(out.n_truncated), int(out.resp_total), int(out.launches))
    for flag in (False, True):
        n_status, n_tc, total, launches = outs[flag]
        print(json.dumps({"ptr": flag, "k": k, "ptr_share": 0.2, "kernel_ms": [round(x, 3) for x in ms[flag]],
                          "best_kernel_ms": round(min(ms[flag]), 3), "queries_per_s": round(k / (min(ms[flag]) / 1e3)),
                          "n_status": n_status, "n_truncated": n_tc, "resp_total": total, "launches": launches,
                          "gpu": gpu, "power_limit_max_sm_clock": power}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
