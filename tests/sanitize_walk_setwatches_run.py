"""TEST INFRASTRUCTURE: small end-to-end run of a watched walk carried across reconnects for compute-sanitizer
(memcheck / racecheck / synccheck): random drop scripts in lockstep with the restatement, from host and device
streams and outputs, then Context.resume_walk end to end.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_walk_setwatches_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import torch
from registrar_b200 import _native
import test_walk_setwatches as t
import walk_setwatches_util as ws

ctx = _native.Context(0)
for seed in range(3):
    rng = random.Random(seed)
    ws.script(rng, t.Lib(ctx, rng), drops=3, depth=3, churn=6, roots=[b"/z", b"/y"], max_frame=[0, 200, 400][seed])
t.test_resume_walk_end_to_end(ctx, 1)
torch.cuda.synchronize()
ctx.close()
print("sanitize_walk_setwatches_run ok")
