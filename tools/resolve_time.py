"""regk_resolve on two device snapshots:
  fleet   4 M config 2 records collapsed onto 1 000 domains (tests/test_mkdirp_set.py's fleet), plus one service record
          per domain: every record of a usable type is a child of its domain's service;
  config3 10 M config 3 records, no service records: HOST_A answers only.
Each is resolved five times (best kernel_ms).  The decode pass is timed on its own by regk_decode over the same device
snapshot (host_nodes = 0, device outputs).  Prints one JSON line per workload with kernel ms, decode ms, launches,
snapshot and text bytes, query and line counts, and the card's name and power limit read in the same run."""
import ctypes as C
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
from registrar_b200.batch import Snapshot

SERVICE = b'{"type":"service","service":{"type":"service","service":{"srvce":"_http","proto":"_tcp","port":80,"ttl":60}}}'


def fleet(n, ndom=1000, seed=3):
    """n config 2 records collapsed onto the domains of the first `ndom`; returns (batch, domain of each record)"""
    rng = np.random.default_rng(seed)
    b = synth.generate("config2", n=n)
    idx = rng.integers(0, ndom, n)
    lens = np.diff(b.domain_off)[idx]
    off = np.zeros(n + 1, np.uint32)
    np.cumsum(lens, out=off[1:])
    pos = np.repeat(b.domain_off[:-1][idx].astype(np.int64) - off[:-1].astype(np.int64), lens) + np.arange(int(off[-1]))
    b.domain_bytes = b.domain_bytes[pos]
    b.domain_off = off
    return b, idx


def snapshot(res, idx):
    """the batch's nodes on the device, followed by one service record per domain when idx is given"""
    pb, po = res.path_bytes[:int(res.path_off[-1])], res.path_off.astype(np.int64)
    jb, jo = res.json_bytes[:int(res.json_off[-1])], res.json_off.astype(np.int64)
    if idx is not None:
        _, first = np.unique(idx, return_index=True)
        dirs = []
        for i in first.tolist():
            p = res.path_bytes[po[i]:po[i + 1]].tobytes()
            dirs.append(p[:p.rfind(b"/")])
        pb = np.concatenate([pb, np.frombuffer(b"".join(dirs), np.uint8)])
        jb = np.concatenate([jb, np.frombuffer(SERVICE * len(dirs), np.uint8)])
        po = np.concatenate([po, po[-1] + np.cumsum([len(d) for d in dirs])])
        jo = np.concatenate([jo, jo[-1] + len(SERVICE) * np.arange(1, len(dirs) + 1)])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return Snapshot(t(pb), t(po), t(jb), t(jo))


def decode_ms(ctx, snap):
    cin, keep = snap.cdecode_in()
    cin.flags |= _native.FLAG_OUT_DEVICE
    out = _native.CDecodeOut()
    ctx._check(ctx._lib.regk_decode(ctx._h, C.byref(cin), C.byref(out)))
    return float(out.kernel_ms)


def measure(ctx, name, batch, idx):
    res = ctx.register_batch(batch)
    snap = snapshot(res, idx)
    del res
    torch.cuda.synchronize()
    runs, dec = [], []
    for _ in range(5):
        t0 = time.perf_counter()
        a = ctx.resolve(snap, 30, 60, device=True)
        runs.append(((time.perf_counter() - t0) * 1e3, float(a.kernel_ms)))
        dec.append(decode_ms(ctx, snap))
    a = ctx.resolve(snap, 30, 60, device=True)
    m = snap.m
    return {"workload": name, "m": m, "snapshot_bytes": snap.path_bytes.numel() + snap.json_bytes.numel() + 16 * (m + 1),
            "text_bytes": int(a.text_total), "queries": int(a.n_queries), "answer_lines": int(a.n_answers),
            "additional_lines": int(a.n_additional), "unresolved": int(a.n_unresolved), "launches": int(a.launches),
            "kernel_ms": [round(k, 3) for _, k in runs], "wall_ms": [round(w, 3) for w, _ in runs],
            "best_kernel_ms": round(min(k for _, k in runs), 3), "best_decode_ms": round(min(dec), 3),
            "best_rest_ms": round(min(k for _, k in runs) - min(dec), 3)}


def main():
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    gpu = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    b, idx = fleet(int(4_000_000 * scale))
    for name, batch, ix in (("fleet", b, idx), ("config3", synth.generate("config3", n=int(10_000_000 * scale)), None)):
        row = measure(ctx, name, batch, ix)
        row.update(gpu=gpu, power_limit_max_sm_clock=power)
        print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
