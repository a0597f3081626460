"""regk_mkdirp_dirs on BASELINE-sized batches: time of the parent pass, the ancestor closure and the gather, set
sizes, and the frames.  Best of 5 calls; one JSON line per case."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from registrar_b200 import _native, synth
from test_mkdirp_set import fleet

ctx = _native.Context(0)
for name, batch in (("config2", synth.generate("config2", n=1_000_000)), ("config3", synth.generate("config3", n=10_000_000)),
                    ("fleet", fleet(4_000_000))):
    ctx.register_batch(batch, copy=False)
    best = None
    for _ in range(5):
        ds = ctx.mkdirp_dirs()
        if best is None or ds.kernel_ms < best.kernel_ms:
            best = ds
    fr = min((ctx.mkdirp_requests() for _ in range(3)), key=lambda f: f[2])
    row = {"case": name, "n": batch.n, "n_dirs": best.n_dirs, "n_invalid": int(best.invalid.size),
           "max_depth": best.max_depth, "dir_bytes": int(best.dir_off[-1]), "launches": best.launches,
           "mkdirp_ms": round(best.kernel_ms, 4), "parent_ms": round(best.parent_ms, 4),
           "closure_ms": round(best.closure_ms, 4), "gather_ms": round(best.gather_ms, 4),
           "frames_ms": round(fr[2], 4), "frame_bytes": int(fr[1][-1])}
    print(json.dumps(row))
ctx.close()
