"""TEST INFRASTRUCTURE: small end-to-end run of regk_walk_resolve for compute-sanitizer (memcheck / racecheck /
synccheck): registry-shaped random scripts with a walk resolve after every refresh, host and device outputs, checked
against the restatement and a plain regk_resolve, then the DNS parity and gate run.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_walk_resolve_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import torch
from registrar_b200 import _native
import test_walk_resolve as t
import walk_resolve_util as wr

ctx, ctx2 = _native.Context(0), _native.Context(0)
for seed in range(3):
    rng = random.Random(seed)
    wr.script(rng, t.Checker(ctx, ctx2, rng), rounds=3, n_svc=3, churn=4, lib=t.ww_lib(ctx, rng))
t.test_dns_answer_parity_and_gate((ctx, ctx2))
torch.cuda.synchronize()
ctx.close()
ctx2.close()
print("sanitize_walk_resolve_run ok")
