"""regk_reconcile on 10 M config 3 records against a device snapshot of the same records with 1 % drift (0.4 % payloads
changed, 0.3 % nodes missing, 0.3 % foreign nodes), in record order and shuffled: wall time and kernel_ms of
regk_reconcile (device outputs) and of each regk_reconcile_requests call, with the card's name and power limit read in
the same run.  The compose step of the same batch is bench.py's ms_per_step (config 3, 10 M); run it in the same call.  Best of 5 (requests: best of 3); one JSON line per case."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from registrar_b200 import _native, synth
from registrar_b200.batch import Snapshot

N = int(os.environ.get("RECONCILE_N", 10_000_000))


def pack(data, off, idx):
    """the slices data[off[i]:off[i+1]] for i in idx, packed, and their u64 offsets"""
    o = off.astype(np.int64)
    lo, lens = o[idx], o[idx + 1] - o[idx]
    noff = np.zeros(idx.size + 1, np.int64)
    np.cumsum(lens, out=noff[1:])
    pos = np.repeat(lo - noff[:-1], lens) + np.arange(int(noff[-1]), dtype=np.int64)
    return data[pos], noff


def snapshot(res, rng, shuffle):
    n = res.n
    pb, po = np.asarray(res.path_bytes), np.asarray(res.path_off)
    jb, jo = np.asarray(res.json_bytes).copy(), np.asarray(res.json_off)
    perm = rng.permutation(n)
    missing, changed, foreign = perm[:n * 3 // 1000], perm[n * 3 // 1000:n * 7 // 1000], perm[n * 7 // 1000:n // 100]
    jb[jo[changed + 1].astype(np.int64) - 1] ^= 1                      # the last payload byte
    keep = np.setdiff1d(np.arange(n), missing)
    kp, ko = pack(pb, po, keep)
    kj, kjo = pack(jb, jo, keep)
    fp, fo = pack(pb, po, foreign)
    fp[fo[1:] - 1] = ord("~")                                           # a path the batch does not have
    fj, fjo = pack(jb, jo, foreign)
    paths = np.concatenate([kp, fp])
    poff = np.concatenate([ko, fo[1:] + ko[-1]])
    datas = np.concatenate([kj, fj])
    joff = np.concatenate([kjo, fjo[1:] + kjo[-1]])
    if shuffle:
        order = rng.permutation(poff.size - 1)
        paths, poff = pack(paths, poff, order)
        datas, joff = pack(datas, joff, order)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return Snapshot(t(paths), t(poff.astype(np.int64)), t(datas), t(joff.astype(np.int64))), (missing.size, changed.size, foreign.size)


def main():
    name = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    batch = synth.generate("config3", n=N)
    res = ctx.register_batch(batch)
    rng = np.random.default_rng(7)
    for shuffle in (False, True):
        snap, drift = snapshot(res, rng, shuffle)
        torch.cuda.synchronize()
        best = None
        for _ in range(5):
            t0 = time.perf_counter()
            d = ctx.reconcile(snap, device=True)
            wall = (time.perf_counter() - t0) * 1e3
            if best is None or wall < best[0]:
                best = (wall, float(d.kernel_ms), d)
        d = best[2]
        row = {"case": "config3 %s" % ("shuffled" if shuffle else "record order"), "n": batch.n, "m": int(d.m),
               "missing": drift[0], "changed": drift[1], "foreign": drift[2],
               "n_same": int(d.n_same), "n_create": int(d.n_create), "n_update": int(d.n_update), "n_delete": int(d.n_delete),
               "launches": int(d.launches), "reconcile_wall_ms": round(best[0], 3), "reconcile_kernel_ms": round(best[1], 3),
               "gpu": name, "power_limit_max_sm_clock": power}
        assert d.n_create == drift[0] and d.n_update == drift[1] and d.n_delete == drift[2]
        for op, label in ((1, "create"), (5, "setdata"), (2, "delete")):
            fr = []
            for _ in range(3):
                t0 = time.perf_counter()
                f = ctx.reconcile_requests(op, device=True)
                fr.append(((time.perf_counter() - t0) * 1e3, float(f.kernel_ms), int(f.total)))
            w, k, tot = min(fr)
            row[label + "_wall_ms"], row[label + "_kernel_ms"], row[label + "_bytes"] = round(w, 3), round(k, 3), tot
        print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
