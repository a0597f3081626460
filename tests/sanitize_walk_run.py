"""TEST INFRASTRUCTURE: small end-to-end run of the registry walk for compute-sanitizer (memcheck / racecheck /
synccheck): a random tree walked from host and device streams with races, errors and notifications, a refused stream
read again once corrected, and the walk's snapshot resolved.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_walk_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import numpy as np
import torch
from registrar_b200 import _native
import test_walk as t
import walk_util as wu

ctx = _native.Context(0)
rng = random.Random(3)
tree = t.random_tree(rng, 4, [0, 1, 5, 40])
for dev_in in (False, True):
    t.run(ctx, tree, [b"/t"], rng, dev_in=dev_in, dev_frames=dev_in,
          knobs=lambda level, frontier: dict(shuffle=True, noise=3, null=True, gd_errors={0: -4}))
ctx.walk_start([b"/t"])
fb = ctx.walk_requests(1)[0]
good = wu.answer(tree, fb, 1)
try:
    ctx.read_walk(np.frombuffer(good[:-5], np.uint8))
    raise AssertionError("a truncated stream was accepted")
except _native.RegkError as e:
    assert e.code == 1
w = ctx.read_walk(t._cuda(good))
ctx.resolve(w, 30, 60)
torch.cuda.synchronize()
ctx.close()
print("sanitize_walk_run ok")
