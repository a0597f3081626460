"""TEST INFRASTRUCTURE: small end-to-end run of REGK_RESOLVE_ANY_FORM for compute-sanitizer (memcheck / racecheck /
synccheck): the README's records verbatim, random mixed snapshots from host and device snapshots with host and device
outputs, a device snapshot ending at its tensor's end, DNS answers after a flagged resolve and the watched README walk.
Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_resolve_any_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch
from registrar_b200 import _native
import test_resolve_any as t

ctx = _native.Context(0)
t.test_readme_records_answer_as_the_readme_shows(ctx)
for seed in range(2):
    t.test_random_mixed_snapshots(ctx, seed)
t.test_device_snapshot_ending_at_the_tensor_end(ctx)
t.test_dns_after_a_flagged_resolve(ctx)
t.test_watched_walk_of_the_readme_tree(True)
torch.cuda.synchronize()
ctx.close()
print("sanitize_resolve_any_run ok")
