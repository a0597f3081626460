"""regk_reconcile against regk_reconcile_owned on 10 M config 3 records and a device snapshot with tools/reconcile_time.py's
drift (0.4 % payloads changed, 0.3 % nodes missing, 0.3 % foreign nodes) plus 1 % of the nodes owned by another session:
kernel_ms of both calls alternated over five rounds (best of 3 within a round), then one REGK_ZK_REPLACE and one
observed-version setData regk_reconcile_requests call (best of 3).  The card's name and power limit are read in the same
run.  One JSON line."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from registrar_b200 import _native, synth
from registrar_b200.batch import Snapshot
from reconcile_time import N, snapshot

SESSION, OTHER = 0x1234_5678_9ABC_DEF0, 0x0FED_CBA9_8765_4321
ROUNDS = 5


def best(fn, k=3):
    out = []
    for _ in range(k):
        t0 = time.perf_counter()
        r = fn()
        out.append(((time.perf_counter() - t0) * 1e3, float(r.kernel_ms if hasattr(r, "kernel_ms") else r.d.kernel_ms), r))
    return min(out, key=lambda x: x[1])


def main():
    name = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    batch = synth.generate("config3", n=N)
    res = ctx.register_batch(batch)
    rng = np.random.default_rng(7)
    snap, drift = snapshot(res, rng, False)
    m = snap.path_off.numel() - 1
    owner = np.full(m, SESSION, np.int64)
    owner[rng.permutation(m)[:m // 100]] = OTHER
    version = rng.integers(-2 ** 31, 2 ** 31, m, dtype=np.int64).astype(np.int32)
    snap = Snapshot(snap.path_bytes, snap.path_off, snap.json_bytes, snap.json_off, torch.from_numpy(version).cuda(),
                    torch.from_numpy(owner).cuda())
    torch.cuda.synchronize()
    plain, owned = [], []
    for _ in range(ROUNDS):
        plain.append(best(lambda: ctx.reconcile(snap, device=True))[1])
        w, k, d = best(lambda: ctx.reconcile_owned(snap, SESSION, device=True))
        owned.append(k)
    row = {"n": batch.n, "m": m, "missing": drift[0], "changed": drift[1], "foreign": drift[2],
           "n_replace": int(d.n_replace), "n_update": int(d.d.n_update), "n_create": int(d.d.n_create),
           "n_delete": int(d.d.n_delete), "launches_owned": int(d.d.launches),
           "reconcile_kernel_ms": [round(x, 3) for x in plain], "reconcile_owned_kernel_ms": [round(x, 3) for x in owned],
           "reconcile_median_ms": round(float(np.median(plain)), 3),
           "reconcile_owned_median_ms": round(float(np.median(owned)), 3)}
    for label, kw in (("replace", dict(op=256, group=1, observed_version=True)),
                      ("setdata_observed", dict(op=5, observed_version=True)),
                      ("setdata", dict(op=5))):
        w, k, f = best(lambda: ctx.reconcile_requests(device=True, **kw))
        row[label + "_wall_ms"], row[label + "_kernel_ms"], row[label + "_bytes"] = round(w, 3), round(k, 3), int(f.total)
    row.update(gpu=name, power_limit_max_sm_clock=power)
    print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
