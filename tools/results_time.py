"""Time regk_read_results on the replies to the single creates of a config 3 first registration, built on the device:
best of five kernel times (CUDA events inside the call), the launch count, and the card it ran on.

    python tools/results_time.py [n] [out.json]      (default n = 10,000,000)
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from registrar_b200 import _native, synth  # noqa: E402
import results_util as su  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    ctx = _native.Context(0)
    res = ctx.register_batch(synth.generate("config3", n=n, seed=5))
    ctx.jute_requests(1, xid_base=1, device=True)
    err = np.where(np.random.default_rng(1).random(n) < 0.01, su.NODEEXISTS, 0).astype(np.int32)
    stream = su.device_create_replies(res.path_bytes, res.path_off, 1, err)
    torch.cuda.synchronize()
    times, launches = [], 0
    for _ in range(6):
        raw = ctx.read_results(stream, _native.RES_BATCH, device=True)
        times.append(float(raw.kernel_ms))
        launches = int(raw.launches)
        assert int(raw.n_failed) == int((err != 0).sum())
    out = dict(card=card, n=n, stream_bytes=int(stream.numel()), best_ms=min(times[1:]), times_ms=times[1:],
               launches=launches)
    print(json.dumps(out))
    if len(sys.argv) > 2:
        with open(sys.argv[2], "w") as f:
            json.dump(out, f)
    ctx.close()


if __name__ == "__main__":
    main()
