"""TEST INFRASTRUCTURE: small end-to-end run of regk_reconcile_owned and of the replace / observed-version frames for
compute-sanitizer (memcheck / racecheck / synccheck), the companion of tests/sanitize_reconcile_run.py: host and device
snapshots with foreign owners, long alias paths, lists whose long-path tiles take the byte-wise framing fallback, a
registry repaired in the model, and the stat refusals.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_reconcile_owned_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import torch
from registrar_b200 import _native, synth
from registrar_b200.batch import RecordBatch, Snapshot
import test_reconcile_owned as t

ctx = _native.Context(0)
paths, pays = t.run(ctx, synth.generate("config3", n=3000, start=5))
t.check_owned(ctx, paths, pays, t.owned_drift(paths, pays, seed=1, frac=0.05, foreign_frac=0.05), groups=(0, 7))
doms = [b"a.b", b"x." * 2500 + b"y", b"q.r"] * 2
paths, pays = t.run(ctx, RecordBatch.from_records(
    [{"domain": d, "hostname": b"h", "type": b"host", "address": b"1.1.1.%d" % i} for i, d in enumerate(doms)], alias=True))
t.check_owned(ctx, paths, pays, [(paths[1], pays[1][:-1], 3, t.OTHER), (paths[1][:-1], b"", -1, t.SESSION)], groups=(0, 1))
paths, pays, nodes = t.fallback_case(ctx)
t.check_owned(ctx, paths, pays, nodes, groups=(0, 100))
paths, pays = t.run(ctx, synth.generate("config3", n=1500, seed=21))
zk, dirs = t._build_registry(paths, pays, random.Random(4))
nodes = t._snapshot(zk, dirs)
t.check_owned(ctx, paths, pays, nodes, groups=(0, 5))
try:
    ctx.reconcile_owned(Snapshot.from_nodes(nodes), 0, 1)
    raise AssertionError("an EPHEMERAL reconcile without a session was accepted")
except _native.RegkError as e:
    assert e.code == 1
torch.cuda.synchronize()
ctx.close()
print("sanitize_reconcile_owned_run ok")
