"""TEST INFRASTRUCTURE: the context-lifetime sequence of tests/test_context_lifetime_gpu.py at a small size for
compute-sanitizer (memcheck / racecheck / synccheck): contexts in a row running every entry-point family, a context
closed with batches in flight on a caller's stream, two contexts with growing shared-memory budgets.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_lifetime_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch
from registrar_b200 import _native
import test_context_lifetime_gpu as t

first = None
for _ in range(2):
    ctx = _native.Context(0)
    got = t.every_family(ctx, n=2200)
    ctx.close()
    first = first or got
assert got == first
t.close_in_flight(n=3000)
t.alternating_budgets(n=1500)
torch.cuda.synchronize()
print("sanitize_lifetime_run ok")
