"""TEST INFRASTRUCTURE: small end-to-end run of regk_children_requests and regk_read_children for compute-sanitizer
(memcheck / racecheck / synccheck), the companion of tests/sanitize_replies_run.py: host and device streams with
notifications, pings, errors, null vectors, a start inside the stream, a stream that ends at its device allocation's
last byte, the stale deletes, and refusals.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_children_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import numpy as np
import torch
from registrar_b200 import _native
from registrar_b200.batch import RecordBatch
import children_util as cu
import test_read_children as t

ctx = _native.Context(0)
paths, pays = t.run(ctx, RecordBatch.from_records(t.fleet_records(2000, 30, seed=3)))
zk = t.drifted(paths, pays, random.Random(1))
fb = t.getchildren(ctx, paths, 2 ** 31 - 10)
stream = cu.replies(zk, fb, errors={5: -4}, null={2}, extra={0: cu.ping(), 9: cu.notification(b"/x" * 40)}, trailing=b"\0\0\0")
t.check(ctx, paths, stream, 2 ** 31 - 10)
t.check(ctx, paths, b"\x01" * 7 + stream, 2 ** 31 - 10, start=7)
exact = torch.from_numpy(np.frombuffer(stream[:-3], np.uint8).copy()).cuda()       # no slack behind the last byte
assert ctx.read_children(exact).n_stale == ctx.read_children(np.frombuffer(stream, np.uint8)).n_stale
ctx.children_requests(t.ZK_DELETE, group=4)
ctx.children_requests(t.ZK_DELETE)
for bad in (stream[:-40], stream[:500] + b"\0\0\0\x05" + stream[500:]):
    try:
        ctx.read_children(np.frombuffer(bad, np.uint8))
        raise AssertionError("a broken stream was accepted")
    except _native.RegkError as e:
        assert e.code == 1
torch.cuda.synchronize()
ctx.close()
print("sanitize_children_run ok")
