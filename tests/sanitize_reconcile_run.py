"""TEST INFRASTRUCTURE: small end-to-end run of regk_reconcile / regk_reconcile_requests for compute-sanitizer
(memcheck / racecheck / synccheck), the companion of tests/sanitize_run.py: host and device snapshots with drift,
duplicates in the batch, an empty snapshot, long alias paths, a dirty skip-mode batch, the tight tables, and the
refusals of a duplicate snapshot path and of corrupt device offsets (refused without a read out of bounds).
Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_reconcile_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch
from registrar_b200 import _native, synth
from registrar_b200.batch import RecordBatch, Snapshot
import test_reconcile as t

ctx = _native.Context(0)
paths, pays = t.run(ctx, synth.generate("config3", n=3000, start=5))
t.check(ctx, paths, pays, t.drift(paths, pays, seed=1, frac=0.05), groups=(0, 7))
t.check(ctx, paths, pays, [], groups=(0,))
recs = [{"domain": b"svc%d.example.com" % (i % 5), "hostname": b"h%d" % (i % 200), "type": b"host",
         "address": b"10.1.1.%d" % i} for i in range(300)]
paths, pays = t.run(ctx, RecordBatch.from_records(recs))
t.check(ctx, paths, pays, list(zip(paths[:80:2], pays[:80:2])))
doms = [b"a.b", b"x." * 2500 + b"y", b"q.r"] * 2
paths, pays = t.run(ctx, RecordBatch.from_records(
    [{"domain": d, "hostname": b"h", "type": b"host", "address": b"1.1.1.%d" % i} for i, d in enumerate(doms)], alias=True))
t.check(ctx, paths, pays, [(paths[1], pays[1][:-1]), (paths[1][:-1], b"")])
base = synth.generate("config3", n=1000, start=9)
dirty = [base.record(i) for i in range(base.n)]
for i in (0, 500, 999):
    dirty[i] = dict(dirty[i], address=b"")
paths, pays = t.run(ctx, RecordBatch.from_records(dirty, types=base.types), skip_bad=True)
t.check(ctx, paths, pays, t.drift(paths, pays, seed=2, frac=0.05))
ctx.set_option("reconcile_tight_table", 1)
t.check(ctx, paths, pays, t.drift(paths, pays, seed=3, frac=0.05))
ctx.set_option("reconcile_tight_table", 0)
nodes = list(zip(paths[:100], pays[:100]))
for snap in (Snapshot.from_nodes(nodes + [nodes[7]]), t.device_snapshot(nodes + [nodes[7]])):
    try:
        ctx.reconcile(snap)
        raise AssertionError("a duplicate snapshot path was accepted")
    except _native.RegkError as e:
        assert e.code == 1 and "node 100 " in e.message
dev = t.device_snapshot(nodes)
po = dev.path_off.clone()
po[50] = dev.path_bytes.numel() + 1000
try:
    ctx.reconcile(Snapshot(dev.path_bytes, po, dev.json_bytes, dev.json_off))
    raise AssertionError("corrupt device offsets were accepted")
except _native.RegkError as e:
    assert e.code == 1 and e.message.endswith("node 49")
torch.cuda.synchronize()
ctx.close()
print("sanitize_reconcile_run ok")
