"""regk_dns_answer on the fleet snapshot of tools/resolve_time.py: 4 M config 2 records collapsed onto 1 000 domains
plus one service record per domain (device snapshot), and device-resident query messages: 60 % host A, 15 % service
SRV, 10 % service A, 15 % AAAA or NX.  Runs: UDP with udp_payload 1232 (10 M queries) and TCP (1 M queries: at the
65535-byte limit every service answer is ~64 KiB, so 10 M of them would not fit in the card's memory).  Each run is one
warm-up and five calls with device outputs (best kernel_ms).  The once-per-resolve preparation is timed on its own: a
one-message call right after the resolve minus the same call again.  Prints one JSON line per run with kernel ms,
queries per second, the bytes read (messages and offsets) and written (responses, offsets and per-message arrays),
status counts, and the card's name and power limit read in the same run."""
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
import dns_util as du


def name_of(path: bytes) -> bytes:
    return b".".join(reversed(path[1:].split(b"/")))


def queries(res, idx, k, rng):
    """k device-resident messages drawn from a pool: (bytes tensor, int64 offsets tensor)"""
    po = res.path_off.astype(np.int64)
    hosts = [name_of(res.path_bytes[po[i]:po[i + 1]].tobytes()) for i in rng.choice(res.n, 50_000, replace=False).tolist()]
    _, first = np.unique(idx, return_index=True)
    svcs = []
    for i in first.tolist():
        p = res.path_bytes[po[i]:po[i + 1]].tobytes()
        svcs.append(name_of(p[:p.rfind(b"/")]))
    groups = [([du.query(h) for h in hosts], 0.60), ([du.query(b"_http._tcp." + s, du.T_SRV, opt=(1232, 0, 0)) for s in svcs], 0.15),
              ([du.query(s) for s in svcs], 0.10),
              ([du.query(h, du.T_AAAA) for h in hosts[:1000]] + [du.query(b"nx%d.example.us" % i) for i in range(1000)], 0.15)]
    pool, weight = [], []
    for msgs, w in groups:
        pool += msgs
        weight += [w / len(msgs)] * len(msgs)
    pick = rng.choice(len(pool), k, p=np.array(weight) / sum(weight))
    lens = np.array([len(x) for x in pool], np.int64)
    starts = np.zeros(len(pool), np.int64)
    np.cumsum(lens[:-1], out=starts[1:])
    off = np.zeros(k + 1, np.int64)
    np.cumsum(lens[pick], out=off[1:])
    blob = torch.from_numpy(np.frombuffer(b"".join(pool), np.uint8).copy()).cuda()
    doff, dpick, dstart = torch.from_numpy(off).cuda(), torch.from_numpy(pick).cuda(), torch.from_numpy(starts).cuda()
    pos = torch.arange(int(off[-1]), device="cuda", dtype=torch.int64)
    which = torch.searchsorted(doff[1:], pos, right=True)
    msgs = blob[dstart[dpick[which]] + pos - doff[which]]
    return msgs, doff


def run(ctx, msgs, off, udp, tcp):
    ctx.answer_dns(msgs, off, udp, tcp, device=True)
    ms = []
    for _ in range(5):
        out = ctx.answer_dns(msgs, off, udp, tcp, device=True)
        ms.append(float(out.kernel_ms))
    k = off.numel() - 1
    read = msgs.numel() + off.numel() * 8
    written = int(out.resp_total) + (k + 1) * 8 + k * (1 + 1 + 8)
    return {"k": k, "tcp": tcp, "udp_payload": udp, "kernel_ms": [round(x, 3) for x in ms], "best_kernel_ms": round(min(ms), 3),
            "queries_per_s": round(k / (min(ms) / 1e3)), "bytes_read": read, "bytes_written": written,
            "resp_total": int(out.resp_total), "n_status": list(out.n_status), "n_truncated": int(out.n_truncated),
            "launches": int(out.launches)}


def main():
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    b, idx = fleet(int(4_000_000 * scale))
    res = ctx.register_batch(b)
    snap = snapshot(res, idx)
    ctx.resolve(snap, 30, 60, device=True)
    one_m, one_o = du.pack([du.query(b"x.example.us")])
    first = ctx.answer_dns(one_m, one_o, device=True)
    again = ctx.answer_dns(one_m, one_o, device=True)
    prep = {"prep_ms": round(float(first.kernel_ms) - float(again.kernel_ms), 3), "m": snap.m,
            "launches_first_call": int(first.launches), "launches_after": int(again.launches), "gpu": gpu,
            "power_limit_max_sm_clock": power}
    print(json.dumps(prep), flush=True)
    rng = np.random.default_rng(7)
    for k, tcp in ((int(10_000_000 * scale), False), (int(1_000_000 * scale), True)):
        msgs, off = queries(res, idx, k, rng)
        row = run(ctx, msgs, off, 1232, tcp)
        row.update(gpu=gpu, power_limit_max_sm_clock=power)
        print(json.dumps(row), flush=True)
        del msgs, off
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
