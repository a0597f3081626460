"""Cost of skip mode (REGK_SKIP_BAD) on device-resident config 3 batches.

Builds are alternated round by round in one process:
  plain        the batch without the flag
  skip-clean   the same clean batch with the flag (expected equal: the same two kernels run)
  skip-1       one record with a bad address byte
  skip-1pct    1 % of the records with a bad address byte
Each call is synchronous (regk_register_batch + regk_finish); the figure is host wall time per call, median over
the rounds.  One extra profiled call per dirty build reports the device time of every kernel by name
(torch.profiler), the skip-mode passes (fence, compact, expand) included.  Prints one JSON object.

    python tools/skip_time.py [--n 10000000] [--rounds 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from registrar_b200 import _native, multigpu, synth  # noqa: E402


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                                       "-i", "0"], text=True).strip()
        return out
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0)


def corrupted(batch, frac, rng):
    """A copy of batch with a '"' as the first address byte of round(frac * n) records (at least one)."""
    b = batch.slice(0, batch.n)
    k = max(1, int(round(frac * b.n)))
    idx = np.sort(rng.choice(b.n, k, replace=False))
    b.addr_bytes[b.addr_off[idx].astype(np.int64)] = ord('"')
    return b, idx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    ctx = _native.Context(0)
    clean = synth.generate("config3", n=a.n)
    ctx.set_types(clean.types)
    rng = np.random.default_rng(1)
    one, _ = corrupted(clean, 0.0, rng)
    pct, idx_pct = corrupted(clean, 0.01, rng)
    builds = {}
    keep = []
    for name, hb, skip in (("plain", clean, False), ("skip-clean", clean, True), ("skip-1", one, True),
                           ("skip-1pct", pct, True)):
        cb, k = multigpu.device_batch(hb, dev)
        keep.append(k)
        builds[name] = (cb, skip)
    torch.cuda.synchronize()
    times = {name: [] for name in builds}
    launches = {}
    for name, (cb, skip) in builds.items():                 # warm-up: allocations, shared-memory attributes
        res = ctx.register_raw(cb, skip_bad=skip)
        launches[name] = int(res.launches)
        if name == "skip-1pct":
            assert ctx.skipped_records()[0].size == idx_pct.size
    for _ in range(a.rounds):
        for name, (cb, skip) in builds.items():
            t0 = time.perf_counter()
            ctx.register_raw(cb, skip_bad=skip)
            times[name].append((time.perf_counter() - t0) * 1e3)
    kernels = {}
    for name in ("skip-clean", "skip-1", "skip-1pct"):
        cb, skip = builds[name]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ctx.register_raw(cb, skip_bad=skip)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t and ("kernel" in ev.key or "Memcpy" in ev.key or "Memset" in ev.key):
                key = ev.key.split("(")[0].replace("void ", "").replace("regk::", "")
                per[key] = round(per.get(key, 0.0) + t / 1e3, 4)
        kernels[name] = per
    out = {"gpu": gpu_info(), "n": a.n, "rounds": a.rounds, "bad_1pct": int(idx_pct.size),
           "ms_median": {k: round(float(np.median(v)), 3) for k, v in times.items()},
           "ms_min": {k: round(float(np.min(v)), 3) for k, v in times.items()},
           "launches": launches, "device_ms_by_kernel": kernels}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
