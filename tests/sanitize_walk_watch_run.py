"""TEST INFRASTRUCTURE: small end-to-end run of the watched walk for compute-sanitizer (memcheck / racecheck /
synccheck): random mutation scripts walked, fed and refreshed in lockstep with the restatement, from host and device
streams, with mutations landing inside reply streams, and the refreshed snapshot resolved.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_walk_watch_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import torch
from registrar_b200 import _native
import test_walk_watch as t
import walk_watch_util as ww

ctx = _native.Context(0)
for seed in range(3):
    rng = random.Random(seed)
    lib = t.Lib(ctx, rng)
    ww.script(rng, lib, rounds=4, depth=3, churn=6, flight=0.2, roots=[b"/z", b"/y"])
    ctx.resolve(lib.w, 30, 60)
torch.cuda.synchronize()
ctx.close()
print("sanitize_walk_watch_run ok")
