"""TEST INFRASTRUCTURE: small end-to-end run of the watched heartbeat for compute-sanitizer (memcheck / racecheck /
synccheck), the companion of tests/sanitize_stats_run.py: watch-byte framings, host and device streams with
notifications, pings and in-range replies, a start inside the stream, a partial trailing frame, a stream that ends at
its device allocation's last byte, the subset exists and getChildren re-checks read back through read_stats,
reconcile_stats and read_children, and refusals.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_events_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import numpy as np
import torch
from registrar_b200 import _native, synth
import events_util as eu
import test_read_events as t

ctx = _native.Context(0)
paths, pays = t.batch(ctx, n=3000, seed=21)
zk = t.watched_model(paths, pays)
t.arm(ctx, zk)
t.drift(zk, paths, pays)
s = zk.take_events(t.SESSION) + t.stream_of(paths, random.Random(3), count=200)
g, _ = t.check(ctx, paths, b"\x01" * 7 + s, start=7, xb=100, nx=50)
exact = torch.from_numpy(np.frombuffer(s + eu.notification(b"/a/b")[:9], np.uint8).copy()).cuda()
assert ctx.read_events(exact, xid_base=100, n_xids=50).partial
ev, st, d, ch = t.period(ctx, zk, 10)
assert d.n_same + d.n_create + d.n_update + d.n_dup + d.n_replace == d.n
t.repair(ctx, zk)
t.period(ctx, zk, 20)
try:
    ctx.read_events(np.frombuffer(s + eu.notification(b"/a", typ=9), np.uint8), xid_base=100, n_xids=50)
    raise AssertionError("a broken stream was accepted")
except _native.RegkError as e:
    assert e.code == 1
torch.cuda.synchronize()
ctx.close()
print("sanitize_events_run ok")
