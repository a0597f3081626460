"""regk_read_replies on 10 M config 3 records: the GetDataResponse stream to the batch's getData frames is built on the
device from the batch (every node found, payload = data, about n x (88 + J) bytes), read back from a device stream five
times (best kernel_ms), then once more under torch.profiler for the per-phase kernel time.  The card's name and power
limit are read in the same run.  One JSON line."""
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
import replies_util as ru

N = 10_000_000
SESSION = 0x1234_5678_9ABC_DEF0
PHASES = (("candidates", ("regk_replies_cand_kernel", "regk_replies_compact_kernel")),
          ("successors_and_jumps", ("regk_replies_succ_kernel", "regk_replies_jump_kernel")),
          ("mark", ("regk_replies_mark_kernel",)),
          ("chain", ("regk_replies_chain_count_kernel", "regk_replies_chain_kernel")),
          ("nodes", ("regk_replies_insert_kernel", "regk_replies_node_count_kernel", "regk_replies_node_kernel")),
          ("gather", ("regk_mkdirp_len_kernel", "regk_mkdirp_gather_kernel")))


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else N
    name = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(0)
    res = ctx.register_batch(synth.generate("config3", n=n))
    ctx.jute_requests(_native.ZK_GETDATA, xid_base=1, device=True)
    rng = np.random.default_rng(7)
    version = rng.integers(0, 100, n, dtype=np.int64).astype(np.int32)
    owner = np.full(n, SESSION, np.int64)
    stream = ru.device_replies(res.json_bytes, res.json_off, 1, version, owner)
    del res
    torch.cuda.synchronize()
    runs = []
    for _ in range(5):
        t0 = time.perf_counter()
        r = ctx.read_replies(stream, device=True)
        runs.append(((time.perf_counter() - t0) * 1e3, float(r.kernel_ms)))
    assert int(r.m) == n and int(r.n_found) == n and int(r.consumed) == stream.numel()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.read_replies(stream, device=True)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        per[ev.key] = per.get(ev.key, 0.0) + ev.device_time_total / 1e3
    phases = {}
    for label, names in PHASES:
        phases[label] = round(sum(v for k, v in per.items() if any(nm in k for nm in names)), 3)
    row = {"n": n, "stream_bytes": stream.numel(), "launches": int(r.launches),
           "kernel_ms": [round(k, 3) for _, k in runs], "wall_ms": [round(w, 3) for w, _ in runs],
           "best_kernel_ms": round(min(k for _, k in runs), 3), "phase_kernel_ms": phases,
           "gpu": name, "power_limit_max_sm_clock": power}
    print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
